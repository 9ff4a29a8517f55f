// Host shim over deepmimic_b200/csrc/kernels/dm_task.cuh for tests/test_task_scenes_cpu.py: the per-environment task-scene logic that
// dm_step_kernel<.., TASK> and dm_task_*_kernel run on the device, compiled here with g++ so it can be checked against the oracle on the CPU.
#include "../deepmimic_b200/csrc/kernels/dm_task.cuh"
#include "../deepmimic_b200/csrc/kernels/dm_task_ext.cuh"

using namespace dmk;

static TaskParams params_from(const double* p) {
    TaskParams P;
    P.timer_min = p[1]; P.timer_max = p[2]; P.max_target_dist = p[3]; P.target_succ_dist = p[4]; P.tar_fail_dist = p[5]; P.pos_reward_scale = p[6];
    P.max_heading_turn_rate = p[7]; P.sharp_turn_prob = p[8]; P.speed_change_prob = p[9]; P.tar_speed_min = p[10]; P.tar_speed_max = p[11]; P.vel_reward_scale = p[12];
    P.tar_speed = p[13]; P.enable_min_tar_vel = static_cast<int>(p[14]); P.pad_ = 0;
    return P;
}

extern "C" {
// p: the 16 doubles of dm_get_task_params (p[0] = kind); t: the environment's task block (kTaskDoubles)
void shim_reset(const double* p, double* t, unsigned long long seed, unsigned long long env, double root_x, double root_z) {
    TaskRng r{seed, env, t + kKCounter};
    task_reset(static_cast<int>(p[0]), params_from(p), t, r, root_x, root_z);
}
void shim_update(const double* p, double* t, unsigned long long seed, unsigned long long env, double dt, double root_x, double root_z) {
    TaskRng r{seed, env, t + kKCounter};
    task_update(static_cast<int>(p[0]), params_from(p), t, r, dt, root_x, root_z);
}
int shim_dist_fail(const double* p, const double* t, double root_x, double root_z) { return task_dist_fail(static_cast<int>(p[0]), params_from(p), t, root_x, root_z) ? 1 : 0; }
void shim_goal(const double* p, const double* t, double root_x, double root_z, double heading, double* out3) { task_goal(static_cast<int>(p[0]), t, root_x, root_z, heading, out3); }
double shim_reward(const double* p, const double* t, int fallen, double root_x, double root_z, double step_dur) {
    return task_reward(static_cast<int>(p[0]), params_from(p), t, fallen != 0, root_x, root_z, step_dur);
}
int shim_task_doubles() { return kTaskDoubles; }
// cSceneImitate::SyncKinCharNewCycle as dm_step_kernel runs it at a clip wrap
void shim_wrap_sync(const double* frame_times, const float* frames, int pose_dim, int num_frames, const float* cycle_delta, double dur, double kin_time,
                    double* origin, double* origin_rot, double sim_x, double sim_z, const double* sim_quat, int sync_pos, int sync_rot) {
    kin_wrap_sync(frame_times, frames, pose_dim, num_frames, cycle_delta, dur, kin_time, origin, origin_rot, sim_x, sim_z, sim_quat, sync_pos != 0, sync_rot != 0);
}

// ---- dm_task_ext.cuh (heading_amp_getup, strike_amp).  xp: 32 doubles = getup_time, heights root / head, recover prob, target_min[3], target_max[3],
// radius, hit reset time, reward scale, hit speed, init hit prob, far prob, near dist, head id, n_strike, strike[4], n_fail, fail[4]
static TaskExtParams ext_from(const double* q) {
    TaskExtParams X;
    X.getup_time = q[0]; X.getup_height_root = q[1]; X.getup_height_head = q[2]; X.recover_episode_prob = q[3];
    for (int k = 0; k < 3; ++k) { X.target_min[k] = q[4 + k]; X.target_max[k] = q[7 + k]; }
    X.target_radius = q[10]; X.hit_reset_time = q[11]; X.tar_reward_scale = q[12]; X.hit_tar_speed = q[13]; X.init_hit_prob = q[14]; X.tar_far_prob = q[15]; X.tar_near_dist = q[16];
    X.head_id = static_cast<int>(q[17]); X.n_strike = static_cast<int>(q[18]);
    for (int k = 0; k < 4; ++k) { X.strike_bodies[k] = static_cast<int>(q[19 + k]); X.fail_bodies[k] = static_cast<int>(q[24 + k]); }
    X.n_fail = static_cast<int>(q[23]);
    return X;
}
// bodies: 38 doubles = head_y, contact_fall, spos[4][3], svel[4][3], fpos[4][3]
static TaskBodies bodies_from(const double* b) {
    TaskBodies B; B.head_y = b[0]; B.contact_fall = static_cast<int>(b[1]);
    for (int k = 0; k < 4; ++k) for (int c = 0; c < 3; ++c) { B.spos[k][c] = b[2 + 3 * k + c]; B.svel[k][c] = b[14 + 3 * k + c]; B.fpos[k][c] = b[26 + 3 * k + c]; }
    return B;
}
void shim_getup_reset(const double* xp, double* x, double kin_time, int clip_is_getup) { getup_reset(ext_from(xp), x, kin_time, clip_is_getup != 0); }
int shim_getup_try_recovery(const double* xp, double* t, unsigned long long seed, unsigned long long env, int test_mode, int terminate_code) {
    TaskRng r{seed, env, t + kKCounter};
    return getup_try_recovery(ext_from(xp), r, test_mode != 0, terminate_code) ? 1 : 0;
}
void shim_getup_recovery_reset(double* t, double* x) { getup_recovery_reset(t, x); }
int shim_getup_update(const double* xp, double* x, double dt, int test_mode, int contact_fall) { return getup_update(ext_from(xp), x, dt, test_mode != 0, contact_fall != 0) ? 1 : 0; }
double shim_getup_phase(const double* xp, const double* x) { return getup_phase(ext_from(xp), x); }
double shim_getup_reward(const double* xp, double root_y, double head_y) { return getup_reward(ext_from(xp), root_y, head_y); }
void shim_strike_reset(const double* p, const double* xp, double* t, double* x, unsigned long long seed, unsigned long long env, double root_x, double root_z, double scene_time, int test_mode) {
    TaskRng r{seed, env, t + kKCounter};
    const TaskParams P = params_from(p);
    task_timer_reset(P, t, r);                                   // cSceneTargetAMP::Reset: the target timer first (SceneTargetAMP.cpp:129-134)
    strike_reset_target(P, ext_from(xp), t, x, r, root_x, root_z, scene_time, test_mode != 0);
    t[kKSpeed] = P.tar_speed; t[kKPrevCom] = t[kKPrevCom + 1] = t[kKPrevCom + 2] = 0.0;
}
void shim_strike_update(const double* p, const double* xp, double* t, double* x, unsigned long long seed, unsigned long long env, double dt, double root_x, double root_z, double scene_time, const double* bodies) {
    TaskRng r{seed, env, t + kKCounter};
    const TaskParams P = params_from(p);
    t[kKTimer] += dt;                                            // cSceneTargetAMP::UpdateTarget without the re-draw (CheckTargetReset is false in this scene)
    strike_update(ext_from(xp), t, x, root_x, root_z, scene_time, bodies_from(bodies));
    if (t[kKTimer] >= t[kKTimerMax]) task_timer_reset(P, t, r);   // cSceneTargetAMP::Update (:136-145)
}
int shim_strike_terminate(const double* p, const double* xp, const double* t, const double* x, double root_x, double root_z, double scene_time) {
    return strike_terminate(params_from(p), ext_from(xp), t, x, root_x, root_z, scene_time);
}
void shim_strike_goal(const double* xp, const double* t, const double* x, double root_x, double root_z, double heading, double scene_time, double* out4) {
    strike_goal(ext_from(xp), t, x, root_x, root_z, heading, scene_time, out4);
}
double shim_strike_reward(const double* p, const double* xp, const double* t, const double* x, int fallen, double root_x, double root_z, double step_dur, int test_mode, int term, double timer_max, double scene_time) {
    return strike_reward(params_from(p), ext_from(xp), t, x, fallen != 0, root_x, root_z, step_dur, test_mode != 0, term, timer_max, scene_time);
}
}

