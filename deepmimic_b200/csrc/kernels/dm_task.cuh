// Per-environment logic of the AMP task scenes, shared by the sm_90a kernels and a host test shim (tests/task_shim.cpp):
//   cSceneTargetAMP   R/DeepMimicCore/scenes/SceneTargetAMP.cpp   goal, reward, target timer / position, distance failure
//   cSceneHeadingAMP  R/DeepMimicCore/scenes/SceneHeadingAMP.cpp  goal, reward, heading / speed random walk
// One thread (lane 0 of the environment's tile) runs these a few times per update, in double like the reference.
// Random draws: the stateless counter stream of the reset kernel, task_u01(seed, global env id, k); the per-environment counter k lives in the
// task block.  cRand::RandDouble(a, a) draws nothing; normal draws are Box-Muller on two consecutive uniforms (DESIGN.md section 8).
#pragma once
#include <cmath>
#include <cstdint>

#if defined(__CUDACC__)
#define DM_HD __host__ __device__ __forceinline__
#else
#define DM_HD inline
#endif

namespace dmk {

enum TaskKind { kTaskNone = 0, kTaskTarget = 1, kTaskHeading = 2, kTaskHeadingGetup = 3, kTaskStrike = 4 };   // 3, 4: dm_task_ext.cuh on top
// the dm_task.cuh behaviour a scene builds on: the get-up scene is a heading scene, the strike scene a target scene
DM_HD int task_base_kind(int kind) { return kind == kTaskHeadingGetup ? kTaskHeading : (kind == kTaskStrike ? kTaskTarget : kind); }

// scene constants (cSceneTargetAMP::ParseArgs SceneTargetAMP.cpp:107-120, cSceneHeadingAMP::ParseArgs SceneHeadingAMP.cpp:71-88)
struct TaskParams {
    double timer_min, timer_max;
    double max_target_dist, target_succ_dist, tar_fail_dist, pos_reward_scale;
    double max_heading_turn_rate, sharp_turn_prob, speed_change_prob, tar_speed_min, tar_speed_max, vel_reward_scale;
    double tar_speed;
    int enable_min_tar_vel, pad_;
};

// TASK block, doubles per environment
constexpr int kTaskDoubles = 16;
enum TaskSlot {
    kKTarX = 0, kKTarZ = 1, kKSpeed = 2, kKHeading = 3, kKTimer = 4, kKTimerMax = 5,
    kKPrevCom = 6,   // 3: COM at the last applied action (cDeepMimicCharController::mPrevActionCOM)
    kKCom = 9,       // 3: COM after the last update of the launch (for CalcReward)
    kKCounter = 12,  // draws consumed so far (exact in a double up to 2^53)
    kKResetSeen = 13 // reset counter of the environment the block was last initialised for
};

// splitmix64 finaliser, the library's one counter-based uniform (reset, task and expert draws), identical to the oracle's U01
DM_HD double task_u01(unsigned long long seed, unsigned long long a, unsigned long long b) {
    unsigned long long z = seed + 0x9E3779B97F4A7C15ull * (a * 2654435761ull + b + 1);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull; z = (z ^ (z >> 27)) * 0x94D049BB133111EBull; z ^= z >> 31;
    return static_cast<double>(z >> 11) * (1.0 / 9007199254740992.0);
}

struct TaskRng {
    unsigned long long seed, env;
    double* counter;   // &task[kKCounter]
    DM_HD double draw() { const unsigned long long k = static_cast<unsigned long long>(*counter); *counter = static_cast<double>(k + 1); return task_u01(seed, env, k); }
    DM_HD double uniform(double lo, double hi) { return (lo == hi) ? lo : lo + draw() * (hi - lo); }   // util/Rand.cpp:30-41
    DM_HD bool coin(double p) { return uniform(0.0, 1.0) < p; }                                          // util/Rand.cpp:137-140
    DM_HD double normal(double mean, double stdev) {                                                     // util/Rand.cpp:50-55
        const double u1 = draw(), u2 = draw();
        return mean + stdev * sqrt(-2.0 * log(1.0 - u1)) * cos(2.0 * 3.14159265358979323846 * u2);
    }
};

DM_HD void task_timer_reset(const TaskParams& P, double* t, TaskRng& r) { t[kKTimer] = 0.0; t[kKTimerMax] = r.uniform(P.timer_min, P.timer_max); }   // util/Timer.cpp:51-69
// cSceneTargetAMP::SampleRandTargetPos (SceneTargetAMP.cpp:259-274)
DM_HD void task_reset_target_pos(const TaskParams& P, double* t, TaskRng& r, double root_x, double root_z) {
    const double dist = r.uniform(0.0, P.max_target_dist);
    const double theta = r.uniform(0.0, 2.0 * 3.14159265358979323846);
    t[kKTarX] = root_x + dist * cos(theta);
    t[kKTarZ] = root_z + dist * sin(theta);
}
DM_HD double task_clamp_speed(int kind, const TaskParams& P, double v) {   // SceneHeadingAMP.cpp:90-94
    return (kind == kTaskHeading) ? fmin(fmax(v, P.tar_speed_min), P.tar_speed_max) : v;
}
// cSceneTargetAMP::Reset after the base reset (SceneTargetAMP.cpp:129-134) + cSceneHeadingAMP::ResetTarget (SceneHeadingAMP.cpp:207-217);
// the controller's ResetParams zeroes mPrevActionCOM (DeepMimicCharController.cpp:227-228)
DM_HD void task_reset(int kind, const TaskParams& P, double* t, TaskRng& r, double root_x, double root_z) {
    task_timer_reset(P, t, r);
    task_reset_target_pos(P, t, r, root_x, root_z);
    if (kind == kTaskHeading) {
        const double speed = r.uniform(P.tar_speed_min, P.tar_speed_max);
        t[kKHeading] = 0.0;
        t[kKSpeed] = task_clamp_speed(kind, P, speed);
    } else {
        t[kKSpeed] = P.tar_speed;
    }
    t[kKPrevCom] = t[kKPrevCom + 1] = t[kKPrevCom + 2] = 0.0;
}
// cSceneTargetAMP::Update after the scene update (SceneTargetAMP.cpp:136-145,232-246) + cSceneHeadingAMP::UpdateTarget (SceneHeadingAMP.cpp:148-205)
DM_HD void task_update(int kind, const TaskParams& P, double* t, TaskRng& r, double dt, double root_x, double root_z) {
    t[kKTimer] += dt;
    if (t[kKTimer] >= t[kKTimerMax]) {
        task_reset_target_pos(P, t, r, root_x, root_z);   // mEnableRandTargetPos stays true in both scenes
        if (kind == kTaskHeading) {
            double delta;
            if (r.coin(P.sharp_turn_prob)) delta = r.uniform(-3.14159265358979323846, 3.14159265358979323846);
            else delta = r.normal(0.0, P.max_heading_turn_rate);
            t[kKHeading] += delta;
            if (r.coin(P.speed_change_prob)) t[kKSpeed] = task_clamp_speed(kind, P, r.uniform(P.tar_speed_min, P.tar_speed_max));
        }
        task_timer_reset(P, t, r);
    }
}
// cSceneTargetAMP::CheckTarDistFail (SceneTargetAMP.cpp:281-292); never in the heading scene (SceneHeadingAMP.cpp:219-222)
DM_HD bool task_dist_fail(int kind, const TaskParams& P, const double* t, double root_x, double root_z) {
    if (kind != kTaskTarget) return false;
    const double dx = root_x - t[kKTarX], dz = root_z - t[kKTarZ];
    return dx * dx + dz * dz > P.tar_fail_dist * P.tar_fail_dist;
}
// cSceneTargetAMP::RecordGoal (SceneTargetAMP.cpp:185-215) / cSceneHeadingAMP::RecordGoal (SceneHeadingAMP.cpp:136-151); heading = cKinTree::CalcHeading
DM_HD void task_goal(int kind, const double* t, double root_x, double root_z, double heading, double* out3) {
    if (kind == kTaskTarget) {
        double rx = t[kKTarX] - root_x, rz = t[kKTarZ] - root_z;
        const double dist = sqrt(rx * rx + rz * rz);
        if (dist > 0.0001) {
            const double c = cos(-heading), s = sin(-heading);   // rotation about +y by -heading (cKinTree::BuildOriginTrans on a direction)
            const double lx = (c * rx + s * rz) / dist, lz = (-s * rx + c * rz) / dist;
            rx = lx; rz = lz;
        } else { rx = 1.0; rz = 0.0; }
        out3[0] = rx; out3[1] = rz; out3[2] = dist;
    } else {
        const double th = t[kKHeading] - heading;
        out3[0] = cos(th); out3[1] = -sin(th); out3[2] = t[kKSpeed];
    }
}
// cSceneTargetAMP::CalcReward (SceneTargetAMP.cpp:3-80) / cSceneHeadingAMP::CalcReward (SceneHeadingAMP.cpp:3-48).
// step_dur = controller time - previous action time; com = t[kKCom], previous = t[kKPrevCom].
DM_HD double task_reward(int kind, const TaskParams& P, const double* t, bool fallen, double root_x, double root_z, double step_dur) {
    if (fallen) return 0.0;
    const double cx = t[kKCom], cz = t[kKCom + 2], px = t[kKPrevCom], pz = t[kKPrevCom + 2];
    if (kind == kTaskTarget) {
        if (task_dist_fail(kind, P, t, root_x, root_z)) return 0.0;
        const double tar_speed = t[kKSpeed];
        const double vel_err_scale = 4.0 / (tar_speed * tar_speed);
        const double dx = t[kKTarX] - root_x, dz = t[kKTarZ] - root_z;
        const double dist_sq = dx * dx + dz * dz;
        const double pos_reward = exp(-P.pos_reward_scale * dist_sq);
        double vel_reward = 0.0;
        if (dist_sq < P.target_succ_dist * P.target_succ_dist) vel_reward = 1.0;
        else {
            const double tx = t[kKTarX] - cx, tz = t[kKTarZ] - cz;
            const double td = sqrt(tx * tx + tz * tz);
            double ux = 0.0, uz = 0.0;
            if (td > 0.0001) { ux = tx / td; uz = tz / td; }
            const double avg_vel = (ux * (cx - px) + uz * (cz - pz)) / step_dur;
            double vel_err = tar_speed - avg_vel;
            if (avg_vel < 0) vel_reward = 0.0;
            else {
                if (P.enable_min_tar_vel) vel_err = fmax(vel_err, 0.0);
                vel_reward = exp(-vel_err_scale * vel_err * vel_err);
            }
        }
        return 0.6 * pos_reward + 0.4 * vel_reward;
    }
    const double h = t[kKHeading];
    const double avg_speed = (cos(h) * (cx - px) - sin(h) * (cz - pz)) / step_dur;
    double vel_reward = 0.0;
    if (avg_speed > 0.0) {
        double vel_err = t[kKSpeed] - avg_speed;
        if (P.enable_min_tar_vel) vel_err = fmax(vel_err, 0.0);
        vel_reward = exp(-P.vel_reward_scale * vel_err * vel_err);
    }
    return vel_reward;
}

// cSceneImitate::SyncKinCharNewCycle (SceneImitate.cpp:420-444) when the looping clip wraps: samples the clip's root at the new mocap time,
// then (sync_rot) RotateRoot -> cKinCharacter::RotateOrigin (KinCharacter.cpp:285-327) with the rotation about +y by (simulated heading -
// kinematic heading), then (sync_pos) moves the origin so the kinematic root's x, z sit on the simulated root and its height offset above the
// (flat, y = 0) ground is kept.  origin: 3 doubles, origin_rot: 4 doubles (w, x, y, z), both in / out.  frames: float pose table with the root
// at [0..2] and its quaternion (w, x, y, z) at [3..6]; sim_quat: the stored world->base quaternion (x, y, z, w) of the simulated character.
DM_HD void kin_wrap_sync(const double* frame_times, const float* frames, int pose_dim, int num_frames, const float* cycle_delta, double dur, double kin_time,
                         double* origin, double* origin_rot, double sim_x, double sim_z, const double* sim_quat, bool sync_pos, bool sync_rot) {
    double org_x = origin[0], org_z = origin[2];
    const int cyc = static_cast<int>(floor(kin_time / dur));
    const double tt = kin_time - cyc * dur;
    int lo = 0, hi = num_frames - 1;   // upper_bound - 1
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (frame_times[mid] <= tt) lo = mid; else hi = mid; }
    double bl = (tt - frame_times[lo]) / (frame_times[lo + 1] - frame_times[lo]);
    bl = fmin(fmax(bl, 0.0), 1.0);
    const float* f0 = frames + static_cast<size_t>(lo) * pose_dim; const float* f1 = f0 + pose_dim;
    const double rx = (1 - bl) * f0[0] + bl * f1[0] + cyc * static_cast<double>(cycle_delta[0]);
    const double rz = (1 - bl) * f0[2] + bl * f1[2] + cyc * static_cast<double>(cycle_delta[2]);
    const double ry = (1 - bl) * f0[1] + bl * f1[1];
    const double qw = origin_rot[0], qx = origin_rot[1], qy = origin_rot[2], qz = origin_rot[3];
    double ux = qy * rz - qz * ry, uy = qz * rx - qx * rz, uz = qx * ry - qy * rx;
    ux *= 2; uy *= 2; uz *= 2;
    double kx = rx + qw * ux + (qy * uz - qz * uy);   // root relative to the origin, rotated by origin_rot
    double kz = rz + qw * uz + (qx * uy - qy * ux);
    if (sync_rot) {
        // kinematic root rotation = origin_rot * slerp(frame roots) (Eigen slerp, shortest arc)
        const double a0 = f0[3], a1 = f0[4], a2 = f0[5], a3 = f0[6], b0 = f1[3], b1 = f1[4], b2 = f1[5], b3 = f1[6];
        const double dq = a0 * b0 + a1 * b1 + a2 * b2 + a3 * b3, ad = fabs(dq);
        double s0, s1;
        if (ad >= 1.0 - 2.220446049250313e-16) { s0 = 1.0 - bl; s1 = bl; }
        else { const double th = acos(ad), sn = sin(th); s0 = sin((1.0 - bl) * th) / sn; s1 = sin(bl * th) / sn; }
        if (dq < 0) s1 = -s1;
        const double cw = s0 * a0 + s1 * b0, cx = s0 * a1 + s1 * b1, cy = s0 * a2 + s1 * b2, cz = s0 * a3 + s1 * b3;
        const double kw = qw * cw - qx * cx - qy * cy - qz * cz, kqx = qw * cx + qx * cw + qy * cz - qz * cy,
                     kqy = qw * cy - qx * cz + qy * cw + qz * cx, kqz = qw * cz + qx * cy - qy * cx + qz * cw;
        // heading = atan2(-z, x) of the rotated +x axis (cKinTree::CalcHeading)
        const double kin_heading = atan2(-2.0 * (kqx * kqz - kw * kqy), 1.0 - 2.0 * (kqy * kqy + kqz * kqz));
        const double bx = -sim_quat[0], by = -sim_quat[1], bz = -sim_quat[2], bw = sim_quat[3];   // root rotation = inverse of world->base
        const double sim_heading = atan2(-2.0 * (bx * bz - bw * by), 1.0 - 2.0 * (by * by + bz * bz));
        const double ha = 0.5 * (sim_heading - kin_heading), dc = cos(ha), ds = sin(ha);           // drot = (dc, 0, ds, 0)
        double nw = dc * qw - ds * qy, nx = dc * qx + ds * qz, ny = dc * qy + ds * qw, nz = dc * qz - ds * qx;   // drot * origin_rot
        const double nn = 1.0 / sqrt(nw * nw + nx * nx + ny * ny + nz * nz);
        origin_rot[0] = nw * nn; origin_rot[1] = nx * nn; origin_rot[2] = ny * nn; origin_rot[3] = nz * nn;
        // origin := root + drot (origin - root); rotation about +y by 2 ha: x' = c x + s z, z' = -s x + c z; y unchanged
        const double c2 = dc * dc - ds * ds, s2 = 2.0 * dc * ds;
        const double wx = org_x + kx, wz = org_z + kz;   // world position of the kinematic root
        org_x = wx + (c2 * (-kx) + s2 * (-kz));
        org_z = wz + (-s2 * (-kx) + c2 * (-kz));
        kx = wx - org_x; kz = wz - org_z;
    }
    if (sync_pos) {
        org_x += sim_x - (kx + org_x);
        org_z += sim_z - (kz + org_z);
        origin[1] = 0.0;   // kin_root.y := ground_h + (kin_root.y - origin.y)  =>  origin.y returns to the ground height 0
    }
    origin[0] = org_x; origin[2] = org_z;
}

}  // namespace dmk
