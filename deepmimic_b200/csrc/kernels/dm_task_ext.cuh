// Per-environment logic of two more AMP task scenes, written as host / device-shared code like dm_task.cuh and checked against the oracle on the
// host (tests/test_task_scenes_cpu.py through tests/task_shim.cpp).  The device glue (what the tile publishes to lane 0 every update in
// dm_step_kernel<.., TASK>, the recovery branch of the reset kernel, the task reset / observe kernels) is checked against the oracle update by
// update on the GPU (tests/test_task_ext_gpu.py).
//   cSceneHeadingAMPGetup  R/DeepMimicCore/scenes/SceneHeadingAMPGetup.cpp  get-up timer, phase goal, get-up reward, recovery episodes
//   cSceneStrikeAMP        R/DeepMimicCore/scenes/SceneStrikeAMP.cpp        point target, hit detection, three-regime reward, success
// Both sit on top of the target / heading logic of dm_task.cuh (task block t, draw stream TaskRng); their own state lives in an extension block x.
#pragma once
#include "dm_task.cuh"

namespace dmk {

constexpr int kMaxTaskBodies = 4;

struct TaskExtParams {
    // cSceneHeadingAMPGetup::ParseArgs (:76-85) + CalcGetupTime (:262-287)
    double getup_time, getup_height_root, getup_height_head, recover_episode_prob;
    // cSceneStrikeAMP::ParseArgs (:212-229)
    double target_min[3], target_max[3];
    double target_radius, hit_reset_time, tar_reward_scale, hit_tar_speed, init_hit_prob, tar_far_prob, tar_near_dist;
    int head_id, n_strike, strike_bodies[kMaxTaskBodies], n_fail, fail_bodies[kMaxTaskBodies];
};

// extension block, doubles per environment
constexpr int kTaskExtDoubles = 8;
enum TaskExtSlot {
    kXTarY = 0,        // strike: target height (x, z are t[kKTarX], t[kKTarZ])
    kXHit = 1,         // strike: mTargetHit
    kXHitTime = 2,     // strike: mTargetHitTime (scene time of the hit, -1 = none)
    kXGetupTimer = 3,  // get-up: mGetupTimer time (its end is getup_time)
    kXNearR = 4,       // strike: near-regime reward term of the current state (max over the strike bodies)
    kXContactFail = 5, // strike: a forbidden body is inside the target sphere
    kXHeadY = 6,       // get-up: height of body head_id after the last update (for CalcRewardGetup at the next query)
    kXRecover = 7      // get-up: the reset kernel started a recovery episode (consumed by the task reset kernel)
};

// what the environment's tile hands to lane 0 after an update: unscaled world positions / COM velocities of a few bodies
struct TaskBodies {
    double head_y;                               // get-up: body head_id
    int contact_fall;                            // cSimCharacter::HasFallen: a fall-contact body touches the ground
    double spos[kMaxTaskBodies][3], svel[kMaxTaskBodies][3];   // strike bodies
    double fpos[kMaxTaskBodies][3];              // bodies that must not touch the target
};

// ------------------------------------------------------------------------------------------------ heading_amp_getup
DM_HD bool getup_active(const TaskExtParams& X, const double* x) { return !(x[kXGetupTimer] >= X.getup_time); }   // CheckGettingUp (:296-299)
// after the scene reset: ResetGetupTimer -> EndGetup, then SyncGetupTimer when the episode starts in a get-up clip (:161-165,179-199)
DM_HD void getup_reset(const TaskExtParams& X, double* x, double kin_time, bool clip_is_getup) { x[kXGetupTimer] = clip_is_getup ? kin_time : X.getup_time; }
// ActivateRecoveryEpisode (:301-317): train mode, a failed episode, a coin from the task stream
DM_HD bool getup_try_recovery(const TaskExtParams& X, TaskRng& r, bool test_mode, int terminate_code) {
    if (!test_mode && X.recover_episode_prob > 0.0 && terminate_code == 1) return r.coin(X.recover_episode_prob);
    return false;
}
// ResetRecoveryEpisode (:40-58): the caller restarts the scene timer and the controller clocks and leaves the character alone; here the
// get-up begins and the controller's previous-action COM is cleared
DM_HD void getup_recovery_reset(double* t, double* x) { x[kXGetupTimer] = 0.0; t[kKPrevCom] = t[kKPrevCom + 1] = t[kKPrevCom + 2] = 0.0; }
// UpdateTimers (:167-171) + UpdateTestGetup (:245-254); returns "getting up" as CheckTerminate / CalcReward of this update see it
DM_HD bool getup_update(const TaskExtParams& X, double* x, double dt, bool test_mode, bool contact_fall) {
    x[kXGetupTimer] += dt;
    if (test_mode && contact_fall && !getup_active(X, x)) x[kXGetupTimer] = 0.0;
    return getup_active(X, x);
}
DM_HD double getup_phase(const TaskExtParams& X, const double* x) { return fmin(fmax(1.0 - x[kXGetupTimer] / X.getup_time, 0.0), 1.0); }   // :289-294
// CalcRewardGetup (:18-38), flat ground at 0
DM_HD double getup_reward(const TaskExtParams& X, double root_y, double head_y) {
    return 0.2 * fmin(fmax(root_y / X.getup_height_root, 0.0), 1.0) + 0.8 * fmin(fmax(head_y / X.getup_height_head, 0.0), 1.0);
}

// ------------------------------------------------------------------------------------------------ strike_amp
DM_HD void strike_set_hit(double* x, bool hit, double scene_time) { if (x[kXHit] == 0.0 && hit) x[kXHitTime] = scene_time; x[kXHit] = hit ? 1.0 : 0.0; }   // :246-255
// ResetTargetPos / Far / Near (:318-374) then ResetTarget's hit initialisation (:300-316,376-383); scene_time = the scene timer (0 at a reset)
DM_HD void strike_reset_target(const TaskParams& P, const TaskExtParams& X, double* t, double* x, TaskRng& r, double root_x, double root_z, double scene_time, bool test_mode) {
    const double pi = 3.14159265358979323846;
    double theta, h, dist;
    if (r.coin(X.tar_far_prob)) { theta = r.uniform(-pi, pi); h = r.uniform(X.target_min[1], X.target_max[1]); dist = r.uniform(X.target_min[2], P.max_target_dist); }
    else { theta = r.uniform(X.target_min[0], X.target_max[0]); h = r.uniform(X.target_min[1], X.target_max[1]); dist = r.uniform(X.target_min[2], X.target_max[2]); }
    strike_set_hit(x, false, scene_time);
    t[kKTarX] = root_x + dist * cos(theta); x[kXTarY] = h; t[kKTarZ] = root_z - dist * sin(theta);
    if (!test_mode && X.init_hit_prob > 0.0) strike_set_hit(x, r.coin(X.init_hit_prob), scene_time);
    x[kXHitTime] = (x[kXHit] != 0.0) ? r.uniform(scene_time - X.hit_reset_time, scene_time) : -1.0;
    x[kXNearR] = 0.0; x[kXContactFail] = 0.0;
}
// UpdateTarget (:289-298) with CheckTargetHit (:440-481); also refreshes the state-dependent pieces CalcReward / CheckTerminate need later
DM_HD void strike_update(const TaskExtParams& X, const double* t, double* x, double root_x, double root_z, double scene_time, const TaskBodies& B) {
    const double tx = t[kKTarX], ty = x[kXTarY], tz = t[kKTarZ], r2 = X.target_radius * X.target_radius;
    double dx = tx - root_x, dz = tz - root_z;
    const double n = sqrt(dx * dx + dz * dz);
    if (n > 1e-5) { dx /= n; dz /= n; } else { dx = 0.0; dz = 0.0; }
    bool hit = false;
    double near_r = 0.0;
    for (int k = 0; k < X.n_strike; ++k) {
        const double ex = tx - B.spos[k][0], ey = ty - B.spos[k][1], ez = tz - B.spos[k][2];
        const double d2 = ex * ex + ey * ey + ez * ez;
        const double speed = dx * B.svel[k][0] + dz * B.svel[k][2];
        if (d2 < r2 && (speed >= X.hit_tar_speed || X.hit_tar_speed == 0.0)) hit = true;
        double vr = fmin(fmax(speed / X.hit_tar_speed, 0.0), 1.0);                       // CalcRewardTargetNear (:72-112)
        vr *= vr;
        near_r = fmax(near_r, 0.2 * exp(-X.tar_reward_scale * d2) + 0.8 * vr);
    }
    if (x[kXHit] == 0.0) strike_set_hit(x, hit, scene_time);
    x[kXNearR] = near_r;
    bool cf = false;                                                                         // CheckTarContactFail (:489-508)
    for (int k = 0; k < X.n_fail; ++k) {
        const double ex = tx - B.fpos[k][0], ey = ty - B.fpos[k][1], ez = tz - B.fpos[k][2];
        if (ex * ex + ey * ey + ez * ez < r2) cf = true;
    }
    x[kXContactFail] = cf ? 1.0 : 0.0;
}
DM_HD double strike_hit_phase(const TaskExtParams& X, const double* x, double scene_time) {   // :390-401
    if (x[kXHit] == 0.0) return 0.0;
    return fmin(fmax((scene_time - x[kXHitTime]) / X.hit_reset_time, 0.0), 1.0);
}
// CheckTerminateTarget (:526-546) after the fall check of the base scene: 0 none, 1 fail, 2 success
DM_HD int strike_terminate(const TaskParams& P, const TaskExtParams& X, const double* t, const double* x, double root_x, double root_z, double scene_time) {
    const double dx = root_x - t[kKTarX], dz = root_z - t[kKTarZ];
    if (dx * dx + dz * dz > P.tar_fail_dist * P.tar_fail_dist) return 1;
    if (x[kXContactFail] != 0.0) return 1;
    if (x[kXHit] != 0.0 && (scene_time - x[kXHitTime]) >= X.hit_reset_time) return 2;
    return 0;
}
// RecordGoal (:407-430): the target in the character's origin frame (origin = root x, z on the ground, rotation about +y by -heading) + hit phase
DM_HD void strike_goal(const TaskExtParams& X, const double* t, const double* x, double root_x, double root_z, double heading, double scene_time, double* out4) {
    const double c = cos(-heading), s = sin(-heading);
    const double lx = t[kKTarX] - root_x, lz = t[kKTarZ] - root_z;
    out4[0] = c * lx + s * lz; out4[1] = x[kXTarY]; out4[2] = -s * lx + c * lz; out4[3] = strike_hit_phase(X, x, scene_time);
}
// CalcReward (:9-190).  Train: hit 1.0; near 0.3 + 0.3 near_r; far 0.3 (0.7 pos + 0.3 vel) and 0 when fallen.  Test: time left at a success.
DM_HD double strike_reward(const TaskParams& P, const TaskExtParams& X, const double* t, const double* x, bool fallen, double root_x, double root_z, double step_dur,
                           bool test_mode, int terminate_code, double timer_max, double scene_time) {
    if (test_mode) return (terminate_code == 2) ? timer_max - scene_time : 0.0;
    if (x[kXHit] != 0.0) return 1.0;
    const double dx = t[kKTarX] - root_x, dz = t[kKTarZ] - root_z, d2 = dx * dx + dz * dz, nd = X.tar_near_dist;
    if (d2 < nd * nd) return 0.3 + 0.3 * x[kXNearR];
    if (fallen) return 0.0;
    const double tar_speed = t[kKSpeed], vel_err_scale = 4.0 / (tar_speed * tar_speed);
    const double rd = sqrt(d2), err = fmax(rd - nd, 0.0);
    const double pos_reward = exp(-P.pos_reward_scale * err * err);
    double vel_reward = 0.0;
    if (rd < nd) vel_reward = 1.0;
    else {
        const double cx = t[kKCom], cz = t[kKCom + 2], px = t[kKPrevCom], pz = t[kKPrevCom + 2];
        const double ux0 = t[kKTarX] - cx, uz0 = t[kKTarZ] - cz, ud = sqrt(ux0 * ux0 + uz0 * uz0);
        double ux = 0.0, uz = 0.0;
        if (ud > 0.0001) { ux = ux0 / ud; uz = uz0 / ud; }
        const double avg_vel = (ux * (cx - px) + uz * (cz - pz)) / step_dur;
        double vel_err = tar_speed - avg_vel;
        if (avg_vel >= 0) { if (P.enable_min_tar_vel) vel_err = fmax(vel_err, 0.0); vel_reward = exp(-vel_err_scale * vel_err * vel_err); }
    }
    return 0.3 * (0.7 * pos_reward + 0.3 * vel_reward);
}

}  // namespace dmk
