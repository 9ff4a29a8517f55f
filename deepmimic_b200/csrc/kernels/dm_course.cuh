// Goal courses of the heading and target scenes: a per-environment list of commanded goals that replaces the scene's own random goals, and
// the record of how closely the character follows it (dm_set_goal_course, dm_get_course_record).  Host / device-shared code like
// dm_latency.cuh: dm_course_kernel (dm_course.cu) runs it on the device, tests/course_shim.cpp on the host against tests/course_ref.py.
//
// Environment e has n_e <= kMaxCoursePoints rows of 3 doubles; n_e = 0 keeps the scene's own goals.
//   heading scenes (heading_amp, heading_amp_getup): rows (t, h, v): the episode time in s (strictly increasing, t_0 >= 0), the heading in
//     radians in task_goal's convention (direction (cos h, -sin h) in the x-z plane, h = 0 along +x) and the speed in m/s.  The goal at
//     episode time tau is row 0 before t_0, the last row from t_{n-1} on, and h, v linear in tau in between; angles are not wrapped.
//   target scene (target_amp): rows (dx, dz, unused): waypoints, offsets in metres from the root's horizontal position when the course
//     started.  Waypoint `active` is the goal; it advances when the root is inside target_succ_dist of it (several in one call if they lie
//     within one radius), and the last one stays the goal once it is reached.  A waypoint further than tar_fail_dist from the character
//     still ends the episode through the scene's own distance failure.
// A course starts at every reset and at dm_set_goal_course: the origin and the previous root are the root now, the previous time the
// episode time now.  After every step launch each course environment (1) writes its record for the interval just stepped, (2) advances its
// waypoints, (3) writes the goal for the new episode time into the task block and (4) parks the scene's redraw timer (kKTimer = 0,
// kKTimerMax = +inf), so the scene draws nothing until the next reset.  In the target scene the record follows the advance, so that it
// counts a waypoint reached at the end of the interval.
// The record, 4 floats:
//   heading: (goal point x, z: 1.5 m from the root along the heading in force during the interval; along-track speed - commanded speed;
//            cross-track speed, positive towards heading h + pi / 2), both speeds the root's horizontal displacement over the interval
//            divided by its episode time, against the goal in force during it; 0 and 0 for an interval of no time
//   target:  (the goal waypoint's x, z; the waypoints reached so far; the root's horizontal distance to the goal waypoint)
#pragma once
#include "dm_task.cuh"

namespace dmk {

constexpr int kMaxCoursePoints = 16;
constexpr int kCourseRecordFloats = 4;
constexpr double kCourseGoalPointDist = 1.5;   // m: the heading record's goal point ahead of the root

// One environment's course and its progress (indexed by environment id)
struct DevCourse {
    int n;        // rows in use; 0: the scene's own goals
    int active;   // target: the goal waypoint, n once the last one has been reached (= the waypoints reached so far)
    int resets;   // the reset counter (kFResets) the course last started at
    int pad_;
    double org_x, org_z;             // the root's horizontal position when the course started
    double prev_x, prev_z, prev_t;   // the root and the episode time at the previous course call
    double row[kMaxCoursePoints][3];
};
static_assert(sizeof(DevCourse) == 440, "DevCourse: four ints, five doubles and 16 rows");

// a + (b - a) w, rounded after each operation (no fused multiply-add), so that the host and the device give the same bits
DM_HD double course_lerp(double a, double b, double w) {
#if defined(__CUDA_ARCH__)
    return __dadd_rn(a, __dmul_rn(__dsub_rn(b, a), w));
#else
    return a + (b - a) * w;
#endif
}

// the heading course's goal at episode time tau
DM_HD void course_heading_goal(const DevCourse& c, double tau, double* h, double* v) {
    const int n = c.n;
    if (tau < c.row[0][0]) { *h = c.row[0][1]; *v = c.row[0][2]; return; }
    if (tau >= c.row[n - 1][0]) { *h = c.row[n - 1][1]; *v = c.row[n - 1][2]; return; }
    int k = 0;
    while (k + 2 < n && tau >= c.row[k + 1][0]) ++k;   // t_k <= tau < t_{k+1}
    const double w = (tau - c.row[k][0]) / (c.row[k + 1][0] - c.row[k][0]);
    *h = course_lerp(c.row[k][1], c.row[k + 1][1], w);
    *v = course_lerp(c.row[k][2], c.row[k + 1][2], w);
}

// the goal waypoint (world x, z) of a target course
DM_HD void course_waypoint(const DevCourse& c, double* wx, double* wz) {
    const int k = c.active < c.n ? c.active : c.n - 1;
    *wx = c.org_x + c.row[k][0];
    *wz = c.org_z + c.row[k][1];
}

// (3) and (4): the goal for episode time tau into the task block, and the scene's redraw timer parked
DM_HD void course_write_goal(int base_kind, const DevCourse& c, double* tk, double tau) {
    if (base_kind == kTaskHeading) course_heading_goal(c, tau, &tk[kKHeading], &tk[kKSpeed]);
    else course_waypoint(c, &tk[kKTarX], &tk[kKTarZ]);
    tk[kKTimer] = 0.0;
    tk[kKTimerMax] = INFINITY;
}

// the record of the interval that ends at (rx, rz, tau), against the goal in the task block (the one in force during it); target courses
// after their advance
DM_HD void course_record(int base_kind, const DevCourse& c, const double* tk, double rx, double rz, double tau, float* rec) {
    if (base_kind == kTaskHeading) {
        const double h = tk[kKHeading], ch = cos(h), sh = sin(h);
        const double dt = tau - c.prev_t;
        double along = 0.0, cross = 0.0;
        if (dt > 0.0) {
            const double dx = rx - c.prev_x, dz = rz - c.prev_z;
            along = (ch * dx - sh * dz) / dt - tk[kKSpeed];
            cross = (-sh * dx - ch * dz) / dt;
        }
        rec[0] = static_cast<float>(rx + kCourseGoalPointDist * ch);
        rec[1] = static_cast<float>(rz - kCourseGoalPointDist * sh);
        rec[2] = static_cast<float>(along);
        rec[3] = static_cast<float>(cross);
    } else {
        double wx, wz;
        course_waypoint(c, &wx, &wz);
        const double dx = rx - wx, dz = rz - wz;
        rec[0] = static_cast<float>(wx);
        rec[1] = static_cast<float>(wz);
        rec[2] = static_cast<float>(c.active);
        rec[3] = static_cast<float>(sqrt(dx * dx + dz * dz));
    }
}

// (2): the waypoints the root (rx, rz) is inside the success radius of, in order
DM_HD void course_advance(const TaskParams& P, DevCourse& c, double rx, double rz) {
    const double r2 = P.target_succ_dist * P.target_succ_dist;
    while (c.active < c.n) {
        const double dx = rx - (c.org_x + c.row[c.active][0]), dz = rz - (c.org_z + c.row[c.active][1]);
        if (!(dx * dx + dz * dz < r2)) break;
        ++c.active;
    }
}

// a course's start at root (rx, rz) and episode time tau (a reset, or dm_set_goal_course): progress, goal, timer and the record of no interval
DM_HD void course_start(int base_kind, DevCourse& c, double* tk, double rx, double rz, double tau, int resets, float* rec) {
    c.active = 0; c.resets = resets;
    c.org_x = rx; c.org_z = rz;
    c.prev_x = rx; c.prev_z = rz; c.prev_t = tau;
    course_write_goal(base_kind, c, tk, tau);
    course_record(base_kind, c, tk, rx, rz, tau, rec);
}

// after a step launch: (1) record, (2) advance (record after it in the target scene), (3) goal, (4) timer
DM_HD void course_step(int base_kind, const TaskParams& P, DevCourse& c, double* tk, double rx, double rz, double tau, float* rec) {
    if (base_kind == kTaskHeading) course_record(base_kind, c, tk, rx, rz, tau, rec);
    else {
        course_advance(P, c, rx, rz);
        course_record(base_kind, c, tk, rx, rz, tau, rec);
    }
    c.prev_x = rx; c.prev_z = rz; c.prev_t = tau;
    course_write_goal(base_kind, c, tk, tau);
}

}  // namespace dmk
