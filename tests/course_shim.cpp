// Host shim over deepmimic_b200/csrc/kernels/dm_course.cuh for tests/test_course_cpu.py: the course rule that dm_course_kernel runs on the
// device, compiled here with g++ so it can be checked against tests/course_ref.py on the CPU.  One course at a time, with its task block.
#include <cstring>

#include "../deepmimic_b200/csrc/kernels/dm_course.cuh"

using namespace dmk;

static DevCourse g_c;
static double g_tk[kTaskDoubles];
static TaskParams g_p;

extern "C" {
int shim_course_bytes() { return static_cast<int>(sizeof(DevCourse)); }
int shim_course_max_points() { return kMaxCoursePoints; }
// base_kind: kTaskHeading (2) or kTaskTarget (1); rows [n x 3]
void shim_course_set(int n, const double* rows, double succ_dist) {
    std::memset(&g_c, 0, sizeof(g_c));
    std::memset(g_tk, 0, sizeof(g_tk));
    std::memset(&g_p, 0, sizeof(g_p));
    g_c.n = n;
    std::memcpy(g_c.row, rows, static_cast<size_t>(n) * 3 * sizeof(double));
    g_p.target_succ_dist = succ_dist;
}
void shim_heading_goal(double tau, double* hv) { course_heading_goal(g_c, tau, &hv[0], &hv[1]); }
void shim_course_start(int kind, double rx, double rz, double tau, float* rec) { course_start(kind, g_c, g_tk, rx, rz, tau, 7, rec); }
void shim_course_step(int kind, double rx, double rz, double tau, float* rec) { course_step(kind, g_p, g_c, g_tk, rx, rz, tau, rec); }
// the task block's goal and timer (kKTarX, kKTarZ, kKSpeed, kKHeading, kKTimer, kKTimerMax) and the progress (active, resets)
void shim_course_state(double* tk6, int* progress2) {
    for (int k = 0; k < 6; ++k) tk6[k] = g_tk[k];
    progress2[0] = g_c.active; progress2[1] = g_c.resets;
}
}
