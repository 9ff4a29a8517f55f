/* deepmimic_b200 -- C ABI of the H100-native batched DeepMimic step.
 *
 * This is the drop-in boundary for the reference's per-step simulation hot path.  Each entry point
 * replaces, for a BATCH of independent environments resident on one GPU, the method of the
 * reference's SWIG-exported facade `cDeepMimicCore` cited next to it (R/ = xbpeng/DeepMimic):
 *
 *   dm_create          cDeepMimicCore(), ParseArgs, Init      R/DeepMimicCore/DeepMimicCore.h:12-25,  DeepMimicCore.cpp:6-54
 *   dm_reset           Reset                                  DeepMimicCore.h:27,                     DeepMimicCore.cpp:61-65
 *   dm_update          Update(timestep)                       DeepMimicCore.h:26,                     DeepMimicCore.cpp:56-59
 *   dm_set_action      SetAction(agent_id, action)            DeepMimicCore.h:58,                     DeepMimicCore.cpp:205-212
 *   dm_record_state    RecordState(agent_id)                  DeepMimicCore.h:56,                     DeepMimicCore.cpp:191-197
 *   dm_record_goal     RecordGoal(agent_id)                   DeepMimicCore.h:57  (size 0 for scene "imitate")
 *   dm_calc_reward     CalcReward(agent_id)                   DeepMimicCore.h:77,                     DeepMimicCore.cpp:327-334
 *   dm_get_flags       NeedNewAction / IsEpisodeEnd / CheckTerminate / CheckValidEpisode
 *                                                             DeepMimicCore.h:55,83-85
 *   dm_get_static      GetStateSize .. BuildActionBoundMax, BuildStateNormGroups   DeepMimicCore.h:62-75
 *   dm_set_mode        SetMode                                DeepMimicCore.h:87
 *   dm_set_sample_count SetSampleCount                        DeepMimicCore.h:88,                     DeepMimicCore.cpp:626-633
 *
 * Plain C: opaque handle, pointers and sizes only, int status (0 = ok) with dm_last_error().  Pointers
 * named d_* are DEVICE pointers (fp32 unless stated), h_* are host pointers.  One host thread per
 * handle; all device work is enqueued on the handle's stream (dm_stream) and is stream-ordered.
 * There is NO CPU fallback: dm_create fails if no CUDA device is usable.
 */
#ifndef DEEPMIMIC_B200_H_
#define DEEPMIMIC_B200_H_
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct dm_handle dm_handle;

typedef struct dm_dims {
    int num_envs;          /* environments simulated by this handle */
    int num_joints;        /* == bodies (15 humanoid3d, 23 dog3d) */
    int pose_dim;          /* DeepMimic pose / vel vector length (43 / 83) */
    int num_dofs;          /* 6 + joint dofs (34 / 70) */
    int state_size;        /* observation length (227 with phase, 226 without, 347 dog) */
    int goal_size;         /* 0 for scene "imitate" */
    int action_size;       /* 28 / 58 */
    int snapshot_size;     /* doubles per env for dm_get_snapshot / dm_set_snapshot */
    int updates_per_action;/* 20 for the shipped arg files (30 Hz queries, 600 Hz updates) */
    int num_update_substeps;
    double motion_duration;
    int amp_obs_size;      /* AMP observation length (226 humanoid3d): GetAMPObsSize, DeepMimicCore.h:78 */
} dm_dims;

enum dm_static_kind {
    DM_STATE_OFFSET = 0, DM_STATE_SCALE = 1, DM_ACTION_OFFSET = 2, DM_ACTION_SCALE = 3,
    DM_ACTION_BOUND_MIN = 4, DM_ACTION_BOUND_MAX = 5, DM_STATE_NORM_GROUPS = 6
};

/* asset_root: directory that contains data/ and args/ (arg-file and asset paths are resolved against it).
 * argv: the reference's argument list, e.g. {"--arg_file", "args/train_humanoid3d_spinkick_args.txt"}.
 * global_env_offset: index of this handle's first env in the whole job (multi-GPU sharding keeps RNG streams independent of the GPU count). */
dm_handle* dm_create(const char* asset_root, int argc, const char** argv, int num_envs, int device, uint64_t seed, uint64_t global_env_offset);
/* Host half of dm_create only (argument files, character / controller / motion loaders, flat model; the work of
 * cDeepMimicCore::ParseArgs + SetupScene's loaders, DeepMimicCore.cpp:40-86): needs no CUDA device.  The handle answers
 * dm_get_dims / dm_get_static / dm_get_model_info; every compute entry point returns an error on it (no CPU fallback). */
dm_handle* dm_load_host(const char* asset_root, int argc, const char** argv);
/* Launch plan of the step kernel for `num_envs` environments on a device with `smem_bytes_per_block` opt-in shared memory per block and `num_sms`
 * multiprocessors (host arithmetic, valid on dm_load_host handles; H100 SXM: 232448 bytes, 132 SMs).  out[9] = {tile width (lanes per environment),
 * environments per block, blocks, dynamic shared memory per block, solver row capacity, floats per environment block, floats of the block-shared
 * tables, offset of the Y block, padded environment count}.  The default configurations are planned as ONE wave (blocks <= SMs). */
int dm_plan_launch(dm_handle* h, int num_envs, int smem_bytes_per_block, int num_sms, int* out9);
enum dm_model_info_kind {
    DM_INFO_PARENTS = 0, DM_INFO_JOINT_TYPES = 1 /* 0 revolute 1 spherical 2 fixed */, DM_INFO_DOF_OFFSETS = 2, DM_INFO_POSE_OFFSETS = 3,
    DM_INFO_FALL_BODIES = 4, DM_INFO_END_EFFECTORS = 5, DM_INFO_LAYOUT = 6 /* {links, 6+dofs, chain stride, tree depth, frames, loop} */
};
/* out: num_joints ints (DM_INFO_LAYOUT: 6 ints).  cKinTree joint-table columns as the kernels see them (anim/KinTree.cpp:25-60). */
int dm_get_model_info(dm_handle* h, int kind, int* out);
/* test hook: 24 doubles per link -- mass, Bullet shape inertia[3], DeepMimic exact inertia[3], pivot->COM[3], parent COM->pivot[3],
 * parent->this rotation (x,y,z,w), revolute axis[3], shape half extents[3], manifold breaking threshold (cSimCharacter::BuildMultiBody,
 * SimCharacter.cpp:789-946, at world scale).  Valid on dm_load_host handles. */
int dm_get_link_table(dm_handle* h, double* h_out);
void dm_destroy(dm_handle* h);
const char* dm_last_error(void);
int dm_get_dims(dm_handle* h, dm_dims* out);
int dm_get_scene_name(dm_handle* h, char* h_out, int capacity);   /* cDeepMimicCore::GetName (DeepMimicCore.cpp:141-150): "Imitate", "Imitate AMP", "Target AMP", ... */
int dm_get_static(dm_handle* h, int kind, double* h_out);   /* h_out: state_size or action_size doubles (norm groups as doubles) */
void* dm_stream(dm_handle* h);                               /* cudaStream_t */
int dm_sync(dm_handle* h);
int dm_set_mode(dm_handle* h, int mode);                     /* 0 train, 1 test (cRLScene::eMode) */
/* Training-sample count of the learner: anneals the episode time limits used by the next resets from (--time_lim_min/max) to
 * (--time_end_lim_min/max) with clamp(count / --anneal_samples, 0, 1)^4 (cRLSceneSimChar::UpdateTimerParams, RLSceneSimChar.cpp:330-347).
 * No-op without --anneal_samples.  Host logic: also valid on dm_load_host handles. */
int dm_set_sample_count(dm_handle* h, long long count);
int dm_set_time_limits(dm_handle* h, double t_min, double t_max);   /* both train-mode bounds directly, bypassing the annealing (measurement / tests) */
int dm_get_time_limits(dm_handle* h, double* h_out3);        /* current train-mode min, max and the test-mode limit (seconds) */

/* Resets the envs whose done flag is set (force_all = 0) or every env (force_all != 0).  Optional host arrays
 * (num_envs doubles each, may be NULL) inject the random draws of the reference's reset: mocap start time,
 * episode time limit, heading rotation -- used by the parity tests to bypass the RNG. */
int dm_reset(dm_handle* h, int force_all, const double* h_kin_time, const double* h_max_time, const double* h_rot_theta);
/* d_actions: [num_envs x action_size] fp32, DeepMimic action layout. */
int dm_set_action(dm_handle* h, const float* d_actions);
/* n_updates consecutive Update(dt) calls in one launch; envs whose episode ended freeze until dm_reset. */
int dm_update(dm_handle* h, double dt, int n_updates);
int dm_record_state(dm_handle* h, float* d_out);             /* [num_envs x state_size] */
int dm_record_goal(dm_handle* h, float* d_out);              /* [num_envs x goal_size] (no-op when goal_size == 0) */
/* AMP task scenes target_amp / heading_amp (cSceneTargetAMP / cSceneHeadingAMP: RecordGoal, CalcReward, target updates; goal_size 3).
 * heading_amp_getup / strike_amp are EXPERIMENTAL (device code written and host-checked, not validated on hardware): dm_create accepts
 * them only with DM_EXPERIMENTAL_TASK_SCENES=1 in the environment.  dm_goal_host is RecordGoal into a host buffer [num_envs x 3]; the task-state hooks
 * expose one environment's task block (16 doubles: target x, z, speed, heading, timer, timer max, previous-action COM[3], COM[3], draw
 * counter, reset counter) and the scene constants + draw-stream key for the parity tests. */
int dm_goal_host(dm_handle* h, float* h_out);
/* Clip datasets (--kin_ctrl clips, cClipsController; task scenes only, experimental like them).  dm_reset_clips = dm_reset with the
 * controller's clip draw injected (h_clip: num_envs ints, may be NULL); dm_record_amp_obs_expert_clips = the expert observation from a given
 * clip per environment (cSceneImitateAMP::SampleExpertMotion); dm_get_clip_table reports the dataset (durations, sampling CDF). */
int dm_reset_clips(dm_handle* h, int force_all, const int* h_clip, const double* h_kin_time, const double* h_max_time, const double* h_rot_theta);
int dm_record_amp_obs_expert_clips(dm_handle* h, const int* h_clip, const double* h_kin_time, float* d_out);
int dm_get_clip_table(dm_handle* h, int* num_clips, double* h_dur, double* h_cdf);
int dm_get_task_state(dm_handle* h, int env, double* h_out16);
int dm_set_task_state(dm_handle* h, int env, const double* h_in16);
int dm_get_task_params(dm_handle* h, double* h_out48, unsigned long long* h_stream2);   /* 16 dm_task.cuh + 32 dm_task_ext.cuh constants */
int dm_calc_reward(dm_handle* h, float* d_out);              /* [num_envs] */
/* cSceneImitate::CalcRewardImitate (SceneImitate.cpp:7-127) whatever the scene's own CalcReward is: in the AMP task scenes it is evaluated
 * against each environment's active clip of the dataset (BASELINE.json config 5: "AMP obs recorded alongside imitate reward"). */
int dm_calc_reward_imitate(dm_handle* h, float* d_out);
/* AMP observations (RecordAMPObsAgent / RecordAMPObsExpert, DeepMimicCore.h:81-82; cSceneImitateAMP::BuildAMPObs): [num_envs x amp_obs_size].
 * Agent: simulated pose / vel now and at the last dm_set_action (call dm_set_action exactly when need_new_action is set, like the
 * reference's agent).  Expert: the clip at h_kin_time[env] (NULL: random U(0, duration) per env and call) and one query period earlier. */
int dm_record_amp_obs_agent(dm_handle* h, float* d_out);
int dm_record_amp_obs_expert(dm_handle* h, const double* h_kin_time, float* d_out);
/* Same with a host output buffer [num_envs x amp_obs_size] (device -> host copy inside); used by the cDeepMimicCore facade. */
int dm_amp_obs_host(dm_handle* h, int expert, const double* h_kin_time, float* h_out);
int dm_observe(dm_handle* h, float* d_state, float* d_reward);  /* fused record_state + calc_reward, either may be NULL */
/* d_flags: [num_envs x 4] int32 = {need_new_action, is_episode_end, check_terminate (0 null / 1 fail), check_valid_episode} */
int dm_get_flags(dm_handle* h, int32_t* d_flags);

/* ---- host-buffer convenience wrappers (the reference-facing plugin path: host in, host out, copies inside).  Page-locked caller buffers
 * (cudaMallocHost / cudaHostRegister) are DMA'd directly; pageable ones pass through the handle's pinned staging buffers. */
int dm_step_host(dm_handle* h, const float* h_actions, double dt, int n_updates, float* h_state, float* h_reward, int32_t* h_flags);
/* Same, and with reset_done != 0 the episodes that ended in this step are restarted (masked dm_reset) after the results have been
 * delivered -- the batched form of the reference caller's "if IsEpisodeEnd(): Reset()" (R/learning/rl_world.py:94-132). */
int dm_step_host_reset(dm_handle* h, const float* h_actions, double dt, int n_updates, float* h_state, float* h_reward, int32_t* h_flags, int reset_done);
/* Measurement hook (bench.py's e2e breakdown): with timing on, every dm_step_host records CUDA events between its phases;
 * dm_step_host_timing returns the last call's {H2D + set_action, update launches, observe + flags, D2H} device ms, then the host's
 * {enqueue, stream-synchronize wait, staging memcpy} wall ms, one spare: 8 doubles. */
int dm_set_timing(dm_handle* h, int on);
int dm_step_host_timing(dm_handle* h, double* h_out8);

/* ---- multi-GPU exchange of the policy step's rows (SURVEY.md 8e: the reference has no multi-GPU path; north_star asks for the step's
 * observations / rewards of all ranks on every rank).  One process per GPU on ONE node, <= 8 ranks.  No collective kernel: every rank's
 * dm_observe_kernel stores its [obs | reward | done] rows straight into the same slots of every peer's buffer (CUDA IPC mapped, NVLink P2P
 * stores from the producing kernel), then raises a per-rank epoch flag in every peer; a consumer waits (on the handle's stream) only when it
 * reads.  Two buffers by step parity: rows of step s may be overwritten by step s + 2 only after every rank released step s, which gives the
 * ranks two steps of slack against each other instead of a barrier per step.
 *   create : allocates the local buffer, returns its 64-byte cudaIpcMemHandle_t; exchange the handles of all ranks (e.g. all_gather_object)
 *   connect: maps the peers (h_ipc_all = world x 64 bytes, own slot ignored)
 *   publish(step): record_state + calc_reward + done of this rank for `step`, stored into every rank's buffer; needs release(step - 2) of all
 *   acquire(step): stream-orders the arrival of every rank's rows of `step`; returns device pointers to [world x N x state], [world x N], [world x N]
 *   release(step): the rows of `step` may be overwritten
 *   status : bit 0 / 1 set if a wait for rows / for a release gave up after 20 s (a peer died) */
int dm_exchange_create(dm_handle* h, int rank, int world, void* h_ipc_out64);
int dm_exchange_connect(dm_handle* h, const void* h_ipc_all);
int dm_exchange_publish(dm_handle* h, long long step);
int dm_exchange_acquire(dm_handle* h, long long step, float** d_obs, float** d_reward, float** d_done);
int dm_exchange_release(dm_handle* h, long long step);
int dm_exchange_status(dm_handle* h, int* status);
int dm_exchange_destroy(dm_handle* h);

/* ---- policy network of the batched rollout on the Hopper tensor cores (SURVEY.md 8(f) rank 1; R/learning/nets/fc_2layers_1024units.py,
 * R/learning/pg_agent.py:140-160, R/learning/normalizer.py): actions = a_mean + a_std * (W2^T relu(W1^T relu(W0^T clip((s - s_mean) / s_std)
 * + b0) + b1) + b2 [+ noise]).  Weights are the reference's dense kernels, [inputs x units] row major, fp32 on the host; they are tiled once
 * into the wgmma operand layout as fp16 hi + lo pairs (exact to fp32 level).  d_obs [rows x in_dim], d_noise [rows x out_dim] or NULL,
 * d_actions [rows x out_dim], all fp32 device pointers; `stream` is a cudaStream_t (e.g. dm_stream(h)); out_dim <= 64. */
typedef struct dm_mlp dm_mlp;
dm_mlp* dm_mlp_create(int device, int in_dim, int h0, int h1, int out_dim, const float* h_w0, const float* h_b0, const float* h_w1, const float* h_b1,
                      const float* h_w2, const float* h_b2, const float* h_in_mean, const float* h_in_std, float in_clip, const float* h_out_mean,
                      const float* h_out_std, int max_rows);
int dm_mlp_forward(dm_mlp* m, const float* d_obs, const float* d_noise, float* d_actions, int rows, void* stream);
long long dm_mlp_launches(dm_mlp* m);
void dm_mlp_destroy(dm_mlp* m);

/* ---- test hooks: raw per-env simulator state, layout shared with the CPU oracle (doubles):
 *  [0..2] basePos(scaled) [3..6] baseQuat world->base (x,y,z,w) [7..9] baseOmega [10..12] baseVel(scaled)
 *  [13 + 4j ..] jointPos(j)  [13 + 4nl + 3j ..] jointVel(j)
 *  [13 + 7nl + (4j+c)*12 ..] manifold point c of link j: valid, localA xyz, worldB xyz, impulse n/t1/t2, distance, lifetime
 *  [13 + 55nl ..] kin_time, origin xyz, origin_rot wxyz, ctrl_time, init_time_offset, prev_action_time, need_new_action, timer, timer_max, 2 spare
 *  [29 + 55nl + 4j ..] PD target of joint j in DeepMimic joint-frame convention (w,x,y,z or angle) */
int dm_get_snapshot(dm_handle* h, int env, double* h_out);
int dm_set_snapshot(dm_handle* h, int env, const double* h_in);
/* profile build only (DM_PROFILE, `make -C deepmimic_b200/csrc profile`; fails in a normal build): per-warp cycle counters by code section of the
 * last dm_update's step kernel, 16 uint32 per warp, block-major ([num_blocks][warps_per_block][16], tools/section_profile.py names them).
 * h_out may be NULL to query the two sizes only. */
int dm_get_section_profile(dm_handle* h, uint32_t* h_out, int* num_blocks, int* warps_per_block);
int dm_get_counters(dm_handle* h, int64_t* h_out);           /* {kernel launches so far, row-capacity overflows seen (must stay 0)} */

#ifdef __cplusplus
}
#endif
#endif
