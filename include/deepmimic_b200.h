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
/* Pushes: a timed external force on one body per environment -- the robustness test of a trained skill (the reference applies such
 * perturbations by hand, one environment at a time, from its viewer).  Host arrays of num_envs entries: h_body [N] (a body / joint id of the
 * character file, -1 = no push), h_force [N x 3] (world axes, the reference's unscaled N), h_start [N] and h_duration [N] (seconds on the
 * environment's episode timer, which every reset sets to 0).  The force acts at the body's COM, times the world scale like gravity, in both
 * Bullet sub-steps of every Update(dt) whose timer value at its start t satisfies start <= t < start + duration; the Stable-PD stage does not
 * see it.  An entry is cleared (body -1) at the end of the update after which t >= start + duration, and by every reset of its environment.
 * dm_set_pushes replaces every entry; it refuses, naming the environment and the argument, a body outside [-1, links), a non-finite force or
 * start, a negative or non-finite duration, and host-only handles.  The first call allocates the handle's push table and switches its step
 * launches to the step kernel's push instantiations; handles that never call it run exactly as before.  Stream-ordered, then synchronises
 * the stream (the staging copy is pageable).  dm_get_pushes writes each environment's current body (-1 when none is pending) to h_body [N].
 * dm_save_state refuses a handle with a pending push; dm_load_state leaves the push table as it is. */
int dm_set_pushes(dm_handle* h, const int32_t* h_body, const float* h_force, const double* h_start, const double* h_duration);
int dm_get_pushes(dm_handle* h, int32_t* h_body);
/* Random pushes for training: a schedule drawn on the device refills every environment's push-table entry (same push semantics as above).
 * h_bodies [n_bodies] (1 to 32 body ids in [0, links)) are the bodies drawn from; force2, duration2 and gap2 are {lo, hi} of the magnitude
 * (N), the duration (s) and the gap after the previous push (s): finite, >= 0, lo <= hi.  At the head of every dm_update a kernel runs, for each
 * real environment whose done flag is clear: when its reset counter has moved since it last ran there, a new episode (draw counter k = 0,
 * last_end = 0); when its entry is empty, five uniforms u = splitmix64(seed ^ "pushes", global env id, k++) in the order gap, body index,
 * magnitude, direction angle a in [0, 2 pi), duration, and the entry becomes body, force (F cos a, 0, F sin a), start = max(last_end + gap,
 * t) with t the episode timer now (a start already passed moves to t), and that duration; last_end = start + duration.  A given global
 * environment gets the same pushes at any GPU count.  The first call allocates the push table and a schedule block of 3 doubles per environment
 * (reset counter seen, k, last_end) and switches the step launches to the push instantiations; later calls replace the parameters.  No host
 * synchronisation per dm_update.  Refused, naming the argument: a body outside [0, links), n_bodies outside [1, 32], a bound that is not
 * finite, negative or with lo > hi, a host-only handle, and a handle with dm_set_pushes tables (dm_set_pushes refuses a scheduled handle).
 * dm_save_state / dm_load_state carry the push table and the schedule block of a scheduled handle; the header's push_schedule field makes a
 * load refuse a blob of a handle with another schedule or none, and the reverse.  Handles without a schedule keep the blob as it was.
 * dm_get_push_table: every environment's entry, body [N], force [N x 3], window [N x 2] (start, duration), and the schedule block [N x 3]
 * (NULL on a handle without a schedule); any pointer may be NULL; synchronises the stream. */
int dm_set_push_schedule(dm_handle* h, const int32_t* h_bodies, int n_bodies, const double* force2, const double* duration2, const double* gap2);
int dm_get_push_table(dm_handle* h, int32_t* h_body, float* h_force, double* h_window, double* h_sched);
/* Per-environment dynamics: every environment e carries 4 + links float factors, friction, kp, kd, torque_limit, then one mass factor per link.
 * The environment steps as the model built from edited asset files would: every PD controller's Kp times kp and Kd times kd, every joint's
 * torque limit times torque_limit, every body's mass times its mass factor (both inertia tensors follow), the contact friction coefficient
 * (0.9 link x 0.9 ground) times friction; the imitation reward's and the task scenes' centre of mass use the environment's masses.
 * Observations are unchanged: the policy is not told the factors.  All factors 1 is the plain model.
 * dm_set_dynamics: explicit factors, h_factors [N x (4 + links)], kept across resets.  friction, kp, kd and torque_limit must be finite and
 * >= 0, a mass factor finite and > 0, and a fixed leaf that the step kernel lumps into its parent (humanoid3d's wrists) must carry its parent's
 * mass factor; a refusal names the environment, the kind and the link.  Stream-ordered, then synchronises the stream.
 * dm_set_dynamics_randomization: lohi [10] = [lo, hi] of friction, kp, kd, torque_limit and mass (finite, >= 0, lo <= hi, mass lo > 0; a
 * refusal names the kind).  Draws every real environment's factors for its current episode, then again at each reset: factor j of the episode
 * with reset counter r is lo + u (hi - lo), u = splitmix64(seed ^ "dynamics", global env id, 64 r + j), j = 0..3 friction, kp, kd,
 * torque_limit, j = 4 + l the mass factor of link l (a lumped leaf copies its parent's).  The same factors at any GPU count.  The first call
 * of either setter allocates the table and synchronises the stream; later randomisation calls and the draws at resets do not.  The table has one owner: each of the two refuses a handle set up by the other.  The first call of either allocates the table
 * and switches the step and observation launches to their dynamics instantiations; handles that never call them run exactly as before.
 * dm_get_dynamics: the factors into d_out [N x (4 + links)] on the device, stream-ordered, no host synchronisation; refuses a handle without a
 * table.  dm_save_state / dm_load_state carry the table of a handle that has one at the end of the blob; the header's dyn_table field makes a
 * load refuse a blob with a table into a handle without one, and the reverse, and its dynamics field (0 without randomisation) a blob of
 * another randomisation or none. */
int dm_set_dynamics(dm_handle* h, const float* h_factors);
int dm_get_dynamics(dm_handle* h, float* d_out);
int dm_set_dynamics_randomization(dm_handle* h, const double* lohi);
/* Control latency: every environment e has a delay d_e, a whole number of updates in [0, updates_per_action - 1] (0-31.7 ms at 600 Hz / 30 Hz).
 * The PD targets of an action set by dm_set_action take effect at the Stable-PD stage of the (d_e + 1)-th update after it; until then the
 * previous targets act.  One action at most is pending per environment: a dm_set_action that arrives while one is still pending replaces it.
 * need_new_action, the AMP history, the task scenes' previous-action COM, observations and rewards stay at the action's time: the policy is not
 * told its delay.  A reset drops the environment's pending action and makes its PD targets the pose the reset wrote, so the first d_e updates
 * of an episode hold the start pose.  d_e = 0 is the plain handle.
 * dm_set_action_latency: h_updates [N] delays, kept across resets; a delay outside [0, updates_per_action - 1] is refused with its environment.
 * Stream-ordered, then synchronises the stream.
 * dm_set_action_latency_randomization: draws every real environment's delay for its current episode, then again at each reset: the delay of the
 * episode with reset counter r is lo + min(hi - lo, floor(u (hi - lo + 1))), u = task_u01(seed ^ "latency", global env id, r), the library's counter-based uniform.  The same
 * delays at any GPU count.  0 <= lo <= hi <= updates_per_action - 1, or a refusal naming the bound.
 * The first call of either setter allocates the table, and every environment that has not run an update of its episode yet (after the handle's
 * own first reset, say) holds its start pose as after a reset; set the table before the episode's first dm_set_action.  That call also
 * switches the action and step launches to their latency instantiations (which also
 * apply the handle's push and dynamics tables), and synchronises the stream; later randomisation calls and the draws at resets do not.  The
 * table has one owner: each of the two refuses a handle set up by the other.  Handles that never call them run exactly as before.
 * dm_get_action_latency: every environment's current delay into d_out [N] on the device, stream-ordered, no host synchronisation; refuses a
 * handle without a table.  dm_save_state / dm_load_state carry the table -- delays, pending targets and the update each takes effect at -- at
 * the end of the blob of a handle that has one, so a save in the middle of a policy step resumes bit for bit; the header's latency_table field
 * makes a load refuse a blob with a table into a handle without one, and the reverse, and the randomisation hash a blob of other bounds or
 * none.  Handles without a table write the blob they wrote before. */
int dm_set_action_latency(dm_handle* h, const int32_t* h_updates);
int dm_set_action_latency_randomization(dm_handle* h, int lo, int hi);
int dm_get_action_latency(dm_handle* h, int32_t* d_out);
/* Goal courses of the heading and target scenes (heading_amp, heading_amp_getup, target_amp): commanded goals instead of the scene's random
 * ones.  Environment e has h_count[e] in [0, 16] rows of 3 doubles at h_rows + e * 16 * 3; a count of 0 keeps the scene's own goals bit for bit.
 *   heading scenes: rows (t, h, v): episode time in s (strictly increasing, t_0 >= 0), heading in radians (direction (cos h, -sin h) in the
 *     x-z plane, h = 0 along +x, the scene's goal convention) and speed in m/s (>= 0).  The goal at episode time tau is row 0 before t_0, the
 *     last row after t_{n-1}, h and v linear in tau in between; angles are not wrapped (0 -> 2 pi is one full turn about +y).
 *   target scene: rows (dx, dz, unused): waypoints, offsets in metres in world axes from the root's horizontal position when the course
 *     started.  The first is the goal; the goal advances when the root comes within the scene's target_succ_dist of it (two waypoints within
 *     one radius both count at once), and the last stays the goal once reached.  A waypoint further than tar_fail_dist from the character
 *     ends the episode through the scene's own distance failure.
 * A course starts at every reset of its environment and at this call: the target origin is the root then, and the goal for the episode time
 * then is in the task block before the next observation.  After every dm_update a course environment records the interval just stepped,
 * advances its waypoints and writes the goal for its new episode time, and the scene's timed redraw never fires (its task draw counter does
 * not move until the next reset).  The step, observation and reward kernels are unchanged: a steered episode's goal observation and reward
 * are the scene's own for the commanded goal.  An environment whose count drops to 0 keeps its last goal until its next reset, where the
 * scene draws its own goals again.  The first call allocates the table; handles that never call it run exactly as before.  The call
 * synchronises the stream; the course launches after resets and updates do not.  Refused by name: a scene without courses, a count outside
 * [0, 16], a row value that is not finite (the target scene's third value is not read), heading times that are not increasing or a negative
 * first time, and a negative speed.  dm_save_state / dm_load_state refuse a handle with a course: courses belong to runs.
 * dm_get_course_record: every environment's record of its last course call into d_out [N x 4] floats on the device, stream-ordered:
 *   heading scenes: (x, z of the point 1.5 m from the root along the heading in force during the interval; along-track speed minus the
 *     commanded speed; cross-track speed, positive towards heading h + pi / 2), the speeds the root's horizontal displacement over the
 *     interval divided by its episode time, 0 for an interval of no time;
 *   target scene: (x, z of the goal waypoint; the waypoints reached so far; the root's horizontal distance to the goal waypoint), after the
 *     call's advance.
 * Environments without a course keep whatever their record last held (zeros at first).  Refused on a handle without a course table. */
int dm_set_goal_course(dm_handle* h, const int32_t* h_count, const double* h_rows);
int dm_get_course_record(dm_handle* h, float* d_out);
/* Placement of the environments in the step kernel (on by default; tile width 16 only, where two environments share a warp: tile width 32
 * handles keep index placement, where it measured slower): every step launch is preceded by a one-block kernel that orders the
 * environments by contact load -- the solver row count of each environment's last Bullet sub-step, its key -- so that environments of equal
 * load share a warp and every block holds its share of heavy warps.  Results are bit-identical either way; off places environment e in tile
 * slot e.  Stream-ordered, no host synchronisation. */
int dm_set_env_order(dm_handle* h, int on);
/* The rule of that placement as host arithmetic (needs no handle or device): order[slot] = environment for slot in [0, n_padded), from
 * keys[n_padded] (padding environments carry the key -1), `tiles` environments of tile width W (16 or 32) per block. */
int dm_plan_env_order(const int* keys, int n_padded, int tiles, int W, int* order);
/* test hook: h_plan3 = {padded environment count, environments per block, tile width}, the keys now (h_keys) and the placement of the last
 * step launch (h_order), padded_envs ints each; any may be NULL.  Synchronises the handle's stream.  The order is the identity when the
 * placement is off. */
int dm_get_env_order(dm_handle* h, int* h_plan3, int* h_keys, int* h_order);
int dm_record_state(dm_handle* h, float* d_out);             /* [num_envs x state_size] */
int dm_record_goal(dm_handle* h, float* d_out);              /* [num_envs x goal_size] (no-op when goal_size == 0) */
/* The simulated character's pose and velocity (cSimCharacter::BuildPose / BuildVel, R/DeepMimicCore/sim/SimCharacter.cpp:1428-1507):
 * [num_envs x pose_dim] fp32 rows in the reference's layout -- root position, root quaternion (w, x, y, z) with w >= 0, then per joint a
 * w-first quaternion (spherical) or the angle wrapped to [-pi, pi] (revolute); the velocity rows hold the root's linear then angular velocity
 * and a 0, then the joints' angular velocities (spherical: 3 and a 0) or rates.  Either pointer may be NULL.  Stream-ordered, no host
 * synchronisation. */
int dm_record_pose(dm_handle* h, float* d_pose, float* d_vel);
/* Rendering of pose rows (the counterpart of the reference's viewer drawing a kin_char, cDrawSceneKinChar / cDrawCharacter, without
 * OpenGL): n_views rows d_pose [n_views x pose_dim] fp32 in dm_record_pose's layout (a motion-file frame; quaternions need not be unit length)
 * are drawn as the handle's character, its collision shapes (box, capsule along the link's y axis, sphere) ray cast on the ground plane
 * y = 0 (a 1 m checker of two greys) under a sky gradient, with one directional light, an ambient term and hard shadows.  One camera for every
 * view, in radians and unscaled metres: it looks at (root x, target_height, root z) of each row from eye = target + distance * (cos pitch sin
 * yaw, sin pitch, cos pitch cos yaw), +y up, fov_y the vertical field of view; one ray per pixel, through its centre.  Outputs (either may
 * be NULL, not both): d_rgb uint8 [n_views x height x width x 3], row 0 at the top; d_ids int16 [n_views x height x width], what each pixel
 * sees: -1 sky, -2 ground, k link k.  Uses the handle's character only, so a handle with num_envs = 1 renders any number of rows.
 * Stream-ordered on the handle's stream, no host synchronisation.  Refused, naming the argument: a host-only handle, n_views outside
 * [1, 65535], width or height outside [16, 4096], a NULL pose, both outputs NULL, a camera value that is not finite, distance <= 0 and
 * fov_y outside (0, pi). */
typedef struct { float yaw, pitch, distance, target_height, fov_y; } dm_camera;
int dm_render_poses(dm_handle* h, int n_views, const float* d_pose, const dm_camera* cam, int width, int height, uint8_t* d_rgb, int16_t* d_ids);
/* dm_render_poses with one marker per view, such as a goal: d_marker [n_views x 4] fp32 (x, y, z, radius) in unscaled metres, a sphere in a
 * colour of its own (green), shaded and shadowed like a link and casting its shadow like one; its pixels have id -3.  A radius <= 0 draws no
 * marker, and a view without one is dm_render_poses's, byte for byte.  Refuses what dm_render_poses refuses and a NULL d_marker. */
int dm_render_poses_marked(dm_handle* h, int n_views, const float* d_pose, const float* d_marker, const dm_camera* cam, int width, int height,
                           uint8_t* d_rgb, int16_t* d_ids);
/* The kinematic character's pose (cKinCharacter::GetPose): [num_envs x pose_dim] fp32 rows in dm_record_pose's layout, every environment's clip
 * sampled at its kin time with the loop's cycle offset and the origin rotation and position applied -- what dm_observe's imitation reward
 * compares against; quaternions with w >= 0.  In --kin_ctrl clips scenes the environment's own clip of the dataset; past the end of a non-looping
 * clip its last frame.  Rows past the real environments are not written; NULL is a no-op.  Stream-ordered, no host synchronisation. */
int dm_record_kin_pose(dm_handle* h, float* d_pose);
/* Tracking error of n episodes: d_a and d_r [T x n x pose_dim] fp32 pose rows in dm_record_pose's layout ([T, N, P]: frame t of episode e at
 * row t n + e), d_len [n] int32 the episodes' lengths in frames.  The feature of a pose is every non-root joint's world origin minus the root's,
 * rotated about y by minus the root's heading; the frame distance d(a, r) is the mean over those joints of the features' Euclidean distance, in
 * metres.  d_lock [n] receives the phase-locked error (1/L) sum_i d(a_i, r_i); d_dtw [n] the time-warped error D(L-1, L-1) / 2L of the DTW
 * recursion over the whole L x L grid, D(0, 0) = 2 d_00, D(i, j) = min(D(i-1, j-1) + 2 d_ij, D(i-1, j) + d_ij, D(i, j-1) + d_ij).  Either output
 * may be NULL.  A length outside [1, T] gives NaN for that episode and reads nothing of it.  Deterministic: an episode's results do not depend
 * on the rest of the batch.  Uses the handle's character only; scratch of (6 (num_joints - 1) + 1) T n floats from the device's stream-ordered
 * memory pool.  Stream-ordered, no host synchronisation.  Refused, naming the argument: a host-only handle, T < 1, n < 1, a NULL input. */
int dm_pose_error(dm_handle* h, int T, int n, const float* d_a, const float* d_r, const int32_t* d_len, float* d_lock, float* d_dtw);
/* AMP task scenes target_amp / heading_amp (cSceneTargetAMP / cSceneHeadingAMP: RecordGoal, CalcReward, target updates; goal_size 3).
 * heading_amp_getup / strike_amp (cSceneHeadingAMPGetup / cSceneStrikeAMP) add a phase to the goal (goal_size 4).  dm_goal_host is RecordGoal
 * into a host buffer [num_envs x goal_size]; the task-state hooks expose one environment's task block (16 doubles: target x, z, speed, heading,
 * timer, timer max, previous-action COM[3], COM[3], draw counter, reset counter, then the 8 doubles of the get-up / strike extension block)
 * and the scene constants + draw-stream key for the parity tests. */
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
/* `rows` (>= 1, any count) expert AMP observations into d_out [rows x amp_obs_size], drawn on the device and enqueued on the handle's stream
 * without a host synchronisation.  Row r draws its clip from the dataset's sampling CDF (task scenes; the scene's motion otherwise) and its
 * time from U(0, clip duration) on the counter stream of (seed, r, call), the call counter advancing once per call; its ground height is
 * environment r % num_envs's.  The rows equal dm_record_amp_obs_expert(_clips) fed the same clips and times.  d_clip_out [rows] int32 and
 * d_time_out [rows] double receive the draws when not NULL.  The draws do not depend on global_env_offset: sharded handles that should draw
 * different rows need different seeds.  dm_expert_sample_count reads (h_get) and then sets (h_set) the call counter; either may be NULL. */
int dm_sample_amp_obs_expert(dm_handle* h, int rows, float* d_out, int* d_clip_out, double* d_time_out);
int dm_expert_sample_count(dm_handle* h, const unsigned long long* h_set, unsigned long long* h_get);
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
/* The goal-conditioned actor of the AMP task scenes (R/learning/nets/fc_2layers_gated_1024units.py:6-58, R/learning/amp_agent.py): with
 * ns = clip((s - s_mean) / s_std), ng = clip((g - g_mean) / g_std), gc = relu(ng Wgc + bgc) and per hidden layer l
 *   gh_l = relu(gc Wgh_l + bgh_l),  h = relu(2 sigmoid(gh_l Wgs_l + bgs_l) * (h W_l + b_l) + gh_l Wgb_l + bgb_l),  h starting as [ns, ng],
 * actions = a_mean + a_std * (h W2 + b2 [+ noise]).  Exactly two hidden layers; gate_common <= 128, gate_hidden <= 64, goal_dim <= 64,
 * out_dim <= 64.  Same weight layout and tiling as dm_mlp_create; the std / mean pointers may be NULL (identity), a clip <= 0 means none. */
typedef struct dm_mlp_gated_weights {
    int in_dim, goal_dim, h0, h1, out_dim, gate_common, gate_hidden;
    const float *w0, *b0, *w1, *b1, *w2, *b2;  /* trunk: [in_dim + goal_dim x h0], [h0 x h1], output layer [h1 x out_dim] */
    const float *gc_w, *gc_b;                  /* gate trunk [goal_dim x gate_common] */
    const float *gh_w[2], *gh_b[2];            /* gate hidden layer l [gate_common x gate_hidden] */
    const float *gs_w[2], *gs_b[2];            /* gate scale of layer l [gate_hidden x h_l] */
    const float *gb_w[2], *gb_b[2];            /* gate bias of layer l [gate_hidden x h_l] */
    const float *s_mean, *s_std, *g_mean, *g_std, *a_mean, *a_std;
    float s_clip, g_clip;
} dm_mlp_gated_weights;
dm_mlp* dm_mlp_create_gated(int device, const dm_mlp_gated_weights* h_weights, int max_rows);
/* d_obs [rows x in_dim], d_goal [rows x goal_dim], d_noise [rows x out_dim] or NULL, d_actions [rows x out_dim]: fp32 device pointers.
 * dm_mlp_forward refuses a gated handle and dm_mlp_forward_gated a plain one. */
int dm_mlp_forward_gated(dm_mlp* m, const float* d_obs, const float* d_goal, const float* d_noise, float* d_actions, int rows, void* stream);
/* The style reward of an AMP agent (Peng et al. 2021, "AMP: Adversarial Motion Priors", eq. 7; R/learning/amp_agent.py): the discriminator is a plain
 * handle from dm_mlp_create with out_dim == 1, the AMP-observation normaliser as its input normaliser and h_out_mean / h_out_std NULL.  Per row r,
 *   d      = W2^T relu(W1^T relu(W0^T clip((x_r - x_mean) / x_std) + b0) + b1) + b2     (the logit, not un-normalised)
 *   style  = max(0, 1 - 0.25 (1 - d)^2)
 *   reward = (1 - task_lerp) style + task_lerp d_task_reward[r],  or style when d_task_reward is NULL.
 * d_amp_obs [rows x in_dim], d_task_reward / d_logit / d_style / d_reward [rows]: fp32 device pointers; d_task_reward, d_logit and d_style may be
 * NULL.  Refused: a gated handle, out_dim != 1, task_lerp outside [0, 1] (or NaN), rows out of range, a NULL d_amp_obs or d_reward. */
int dm_mlp_forward_style_reward(dm_mlp* m, const float* d_amp_obs, const float* d_task_reward, float task_lerp, float* d_logit, float* d_style, float* d_reward,
                                int rows, void* stream);
long long dm_mlp_launches(dm_mlp* m);   /* kernel launches so far: 4 per plain forward, 6 per gated forward, 4 per style-reward forward */
void dm_mlp_destroy(dm_mlp* m);
/* PPO value targets of a rollout window (R/learning/rl_util.py: compute_return, R/learning/ppo_agent.py: _compute_batch_vals), one launch.
 * The critic is a dm_mlp handle with out_dim == 1 and the value normaliser as its output normaliser (plain: dm_mlp_create; goal-conditioned:
 * dm_mlp_create_gated).  Inputs [T x N] row major (step k, environment n at k N + n): d_rewards, d_values = V(s_k), d_end_values = V(s'_k) with
 * s'_k the state after step k before the reset, d_done (0 / 1 bytes), d_terminate (0 null, 1 fail, 2 succ).  Per environment, k = T - 1 .. 0:
 *   v_next = done[k] ? (terminate[k] == 1 ? val_fail : terminate[k] == 2 ? val_succ : end_values[k]) : end_values[k]
 *   G_next = (done[k] || k == T - 1) ? v_next : returns[k + 1]
 *   returns[k] = rewards[k] + discount ((1 - td_lambda) v_next + td_lambda G_next),   advantages[k] = returns[k] - values[k]   (fp32)
 * A path still running at step T - 1 is bootstrapped with V(s'_{T-1}), as a null end is.  Refused: T or N <= 0, discount outside [0, 1),
 * td_lambda outside [0, 1] (either NaN), a NULL pointer. */
int dm_td_lambda_returns(const float* d_rewards, const float* d_values, const float* d_end_values, const uint8_t* d_done, const int32_t* d_terminate, int T, int N,
                         float discount, float td_lambda, float val_fail, float val_succ, float* d_returns, float* d_advantages, void* stream);
/* Re-tiles a plain handle's weights from fp32 DEVICE memory, [units x inputs] row major (the transpose of dm_mlp_create's layout: d_w0 [h0 x in_dim], d_w1 [h1 x h0],
 * d_w2 [out_dim x h1], biases [units]) on `stream`, without a host round trip: the same tiles dm_mlp_create builds from the transposed weights.
 * The normalisers are kept.  Refused: a NULL handle or pointer, a gated handle. */
int dm_mlp_set_weights_device(dm_mlp* m, const float* d_w0, const float* d_b0, const float* d_w1, const float* d_b1, const float* d_w2, const float* d_b2,
                              void* stream);

/* Refreshes a plain handle's normalisers from fp32 DEVICE statistics on `stream`: d_in_mean / d_in_std [in_dim] (the handle keeps 1 / std, as
 * dm_mlp_create does), d_out_mean / d_out_std [out_dim].  The same values dm_mlp_create would store.  Refused: a NULL handle or pointer, a gated
 * handle. */
int dm_mlp_set_normalizers_device(dm_mlp* m, const float* d_in_mean, const float* d_in_std, const float* d_out_mean, const float* d_out_std, void* stream);

/* ---- PPO minibatch step of a plain 2-layer network on the Hopper tensor cores (R/learning/ppo_agent.py: PPOAgent._update_actor /
 * _update_critic; solvers/mpi_solver.py wrapping TF's MomentumOptimizer).  A dm_learn workspace holds a learner-owned dm_mlp handle of
 * max_rows rows (the forward's saved activations), the backward operand tiles and the dW partials.  kind 0: the PPO actor (out_dim <= 64
 * normalised action means), kind 1: the critic (out_dim 1, the normalised value).  The parameters are the caller's fp32 device tensors in
 * [units x inputs] layout of dm_mlp_set_weights_device and are updated in place, with the caller's momentum accumulators of the same shapes. */
typedef struct dm_learn dm_learn;
typedef struct dm_learn_net {
    float *w[3], *b[3];            /* parameters: w[l] [units x inputs], b[l] [units] */
    float *acc_w[3], *acc_b[3];    /* momentum accumulators, same shapes */
} dm_learn_net;
/* One minibatch of `rows` rows of a window of samples.  Per row r with sample s = idx[r]:
 *   x = clip((states[s] - in_mean) * in_istd, +-in_clip) through the network: y = the normalised output.
 *   actor:  logp = sum_j (-0.5 ((norm_actions[s][j] - y_j) / sigma_j)^2 - logstd[j] - 0.5 log(2 pi)),  sigma = exp(logstd),
 *           ratio = exp(logp - old_logp[s]) (written to ratio[r] when ratio is not NULL),  A = adv[s],
 *           loss = -mean_r min(A ratio, A clip(ratio, 1 +- ratio_clip)) + 0.5 mean_r sum_j (min(y_j - bound_min_j, 0)^2 + max(y_j - bound_max_j, 0)^2);
 *           the surrogate's gradient flows where the unclipped term is the minimum (ties included) or the ratio lies inside the clip range.
 *           stats[0] += |loss|, stats[1] += the fraction of rows with |ratio - 1| > ratio_clip.
 *   critic: loss = 0.5 mean_r (norm_targets[s] - y)^2;  stats[0] += loss.
 * Then per parameter g = dloss/dw + weight_decay w (weights only), acc = momentum acc + g, w -= stepsize acc.  The step is bit-reproducible
 * (fixed-order reductions).  fp32 device pointers except idx (int64); the actor-only pointers may be NULL for the critic and targets for the
 * actor. */
typedef struct dm_learn_batch {
    const float* states;           /* [samples x in_dim] */
    const int64_t* idx;            /* [rows] */
    int rows;
    const float *in_mean, *in_istd;
    float in_clip;                 /* <= 0: none */
    const float *norm_actions, *old_logp, *adv, *logstd, *bound_min, *bound_max;   /* actor: [samples x out_dim], [samples], [samples], [out_dim] x 3 */
    float ratio_clip;
    float* ratio;                  /* actor, optional: [rows] the probability ratio of every row */
    const float* norm_targets;     /* critic: [samples] */
    float stepsize, momentum, weight_decay;
    float* stats;                  /* actor: 2 floats, critic: 1 */
} dm_learn_batch;
/* kind 2: the AMP discriminator (R/learning/amp_agent.py: AMPAgent._build_losses, _disc_grad_penalty_loss, _disc_weight_decay_loss,
 * _disc_logit_reg_loss, _update_disc), out_dim 1, stepped by dm_learn_disc_step; max_rows counts the rows of one step, agent and expert
 * together (up to max_rows / 2 per side).  One step of `rows` agent rows a_r = agent[agent_idx[r]] and `rows` expert rows
 * e_r = expert[expert_idx[r]], each normalised and clipped as x = clip((. - in_mean) * in_istd, +-in_clip), logits d = D(x):
 *   disc_loss    = 0.5 (0.5 mean_r (d(e_r) - 1)^2 + 0.5 mean_r (d(a_r) + 1)^2)              (least squares, Peng et al. 2021, eq. 8)
 *   grad_penalty = 0.5 mean_r ||dd/dx (e_r)||^2                                                (the ReLU masks held constant)
 *   loss = disc_loss + grad_penalty_weight grad_penalty + weight_decay sum_l ||W_l||^2 / 2 (the logit layer included, biases not)
 *          + logit_reg_weight ||W_logit||^2 / 2
 * then acc = momentum acc + dloss/dw, w -= stepsize acc.  stats (6 floats) += {disc_loss, grad_penalty, mean(d_e > 0), mean(d_a < 0), mean d_e,
 * mean d_a}.  Bit-reproducible (fixed-order reductions).  fp32 device pointers except the int64 indices. */
typedef struct dm_learn_disc_batch {
    const float *agent, *expert;   /* [agent samples x in_dim], [expert samples x in_dim] */
    const int64_t *agent_idx, *expert_idx;   /* [rows] each */
    int rows;                      /* per side */
    const float *in_mean, *in_istd;
    float in_clip;                 /* <= 0: none */
    float stepsize, momentum, weight_decay, logit_reg_weight, grad_penalty_weight;
    float* stats;                  /* 6 floats */
} dm_learn_disc_batch;
/* Refused: no CUDA device or not sm_90a, a kind other than 0, 1, 2, bad sizes (out_dim <= 64, kinds 1 and 2 need out_dim 1), max_rows <= 0
 * (kind 2: < 2). */
dm_learn* dm_learn_create(int device, int kind, int in_dim, int h0, int h1, int out_dim, int max_rows);
/* Loads the parameters' current values into the workspace's tiles (call before the first step and whenever they changed elsewhere). */
int dm_learn_set_weights(dm_learn* l, const dm_learn_net* net, void* stream);
/* One PPO minibatch step (kinds 0 and 1), 15 launches on `stream`.  Refused: a NULL handle or pointer, a kind 2 workspace, rows outside
 * [1, max_rows], ratio_clip <= 0, a negative stepsize, momentum or weight_decay (or NaN). */
int dm_learn_step(dm_learn* l, const dm_learn_net* net, const dm_learn_batch* batch, void* stream);
/* One discriminator step (kind 2), 26 launches on `stream`.  Refused: a NULL handle or pointer, a kind 0 or 1 workspace, rows outside
 * [1, max_rows / 2], a negative (or NaN) stepsize, momentum, weight_decay, logit_reg_weight or grad_penalty_weight. */
int dm_learn_disc_step(dm_learn* l, const dm_learn_net* net, const dm_learn_disc_batch* batch, void* stream);
/* PPO minibatch steps of the gated networks of the AMP task scenes (fc_2layers_gated_1024units, dm_mlp_create_gated's network): kind 0 the
 * actor, kind 1 the critic (out_dim 1).  Same rules, losses and statistics as dm_learn_step; the input is [normalised state | normalised goal]
 * and the goal alone feeds the gates.  Ten parameter pairs in [units x inputs] layout (dm_learn_net's), in this order: the trunk W0 [h0 x (in_dim +
 * goal_dim)], W1 [h1 x h0], the output layer W2 [out_dim x h1], the gate trunk Wgc [gate_common x goal_dim], the gate hidden layers Wgh_0,
 * Wgh_1 [gate_hidden x gate_common], the gate scales Ws_0 [h0 x gate_hidden], Ws_1 [h1 x gate_hidden] and the gate biases Wt_0, Wt_1 (same
 * shapes as the scales); each bias [units]. */
typedef struct dm_learn_gated_net {
    float *w[10], *b[10];
    float *acc_w[10], *acc_b[10];
} dm_learn_gated_net;
/* batch: as for dm_learn_step; goals [samples x goal_dim] (row idx[r] of every minibatch row r), normalised as clip((g - g_mean) * g_istd,
 * +-g_clip) (g_clip <= 0: none). */
typedef struct dm_learn_gated_batch {
    dm_learn_batch batch;
    const float* goals;
    const float *g_mean, *g_istd;
    float g_clip;
} dm_learn_gated_batch;
/* Refused: no CUDA device or not sm_90a, a kind other than 0, 1, a critic with out_dim != 1, the sizes dm_mlp_create_gated refuses
 * (goal_dim <= 64, gate_common <= 128, gate_hidden <= 64, out_dim <= 64), max_rows <= 0. */
dm_learn* dm_learn_create_gated(int device, int kind, int in_dim, int goal_dim, int h0, int h1, int out_dim, int gate_common, int gate_hidden, int max_rows);
/* dm_learn_set_weights and dm_learn_step of a gated workspace (32 launches per step); each refuses a plain workspace, and the plain functions
 * refuse a gated one. */
int dm_learn_set_gated_weights(dm_learn* l, const dm_learn_gated_net* net, void* stream);
int dm_learn_gated_step(dm_learn* l, const dm_learn_gated_net* net, const dm_learn_gated_batch* batch, void* stream);
/* Re-tiles a dm_mlp_create_gated handle from fp32 DEVICE weights d_w[10], d_b[10] in dm_learn_gated_net's order and layout, and refreshes its
 * state, goal and output normalisers from device statistics ([in_dim], [goal_dim], [out_dim]; the handle keeps 1 / std of the first two), on
 * `stream`: the values dm_mlp_create_gated stores.  Refused: a NULL handle or pointer, a plain handle. */
int dm_mlp_set_gated_weights_device(dm_mlp* m, const float* const* d_w, const float* const* d_b, void* stream);
int dm_mlp_set_gated_normalizers_device(dm_mlp* m, const float* d_s_mean, const float* d_s_std, const float* d_g_mean, const float* d_g_std, const float* d_out_mean,
                                        const float* d_out_std, void* stream);
/* The minibatch step split in two around its gradient, for data-parallel training (solvers/mpi_solver.py: MPISolver averages the workers' flat
 * gradients before the momentum step).  Between the halves the caller may sum the ranks' buffers (e.g. one all-reduce).
 *   dm_learn_grad_size: the floats of the network's flat gradient (-1 on a NULL handle): per parameter pair, in the order of the net struct
 *     (dm_learn_net: layers 0, 1, 2; dm_learn_gated_net: its ten pairs), the weights [units x inputs] row major, then the bias [units].
 *     For the gated networks this is not the Python modules' parameter order (capi.py: gated_layers() gives the pairs in this order, and
 *     TensorCoreLearner.grad_views() maps the buffer to the parameters).
 *   *_grad: the step's launches up to its layer pass (the same forward, head, backward and statistics: `stats` accumulates as in the step),
 *     then one pack pass that writes the mean gradient over the step's rows into d_grad: the split-K partials summed in the step's order, times
 *     1 / rows, plus (discriminator) the weighted penalty's.  Without weight decay and the logit regulariser: they depend on the weights alone.
 *     The parameters are read only.  Same launch count as the step.
 *   *_apply: the layer pass on g = scale * d_grad: weight decay (and the logit regulariser) added, the momentum step and the re-tiling, one
 *     launch per parameter pair.  Reads the batch's stepsize, momentum, weight_decay (and logit_reg_weight) only.
 * apply(grad(b), scale 1) leaves the parameters, accumulators, tiles and statistics bit-identical to the step on b.  Refused: a NULL handle or
 * pointer, the wrong workspace kind, what the step refuses (grad), a negative (or NaN) optimiser field or a non-finite scale (apply). */
long long dm_learn_grad_size(const dm_learn* l);
int dm_learn_grad(dm_learn* l, const dm_learn_net* net, const dm_learn_batch* batch, float* d_grad, void* stream);
int dm_learn_apply(dm_learn* l, const dm_learn_net* net, const dm_learn_batch* batch, const float* d_grad, float scale, void* stream);
int dm_learn_gated_grad(dm_learn* l, const dm_learn_gated_net* net, const dm_learn_gated_batch* batch, float* d_grad, void* stream);
int dm_learn_gated_apply(dm_learn* l, const dm_learn_gated_net* net, const dm_learn_gated_batch* batch, const float* d_grad, float scale, void* stream);
int dm_learn_disc_grad(dm_learn* l, const dm_learn_net* net, const dm_learn_disc_batch* batch, float* d_grad, void* stream);
int dm_learn_disc_apply(dm_learn* l, const dm_learn_net* net, const dm_learn_disc_batch* batch, const float* d_grad, float scale, void* stream);
void dm_learn_destroy(dm_learn* l);

/* ---- test hooks: raw per-env simulator state, layout shared with the CPU oracle (doubles):
 *  [0..2] basePos(scaled) [3..6] baseQuat world->base (x,y,z,w) [7..9] baseOmega [10..12] baseVel(scaled)
 *  [13 + 4j ..] jointPos(j)  [13 + 4nl + 3j ..] jointVel(j)
 *  [13 + 7nl + (4j+c)*12 ..] manifold point c of link j: valid, localA xyz, worldB xyz, impulse n/t1/t2, distance, lifetime
 *  [13 + 55nl ..] kin_time, origin xyz, origin_rot wxyz, ctrl_time, init_time_offset, prev_action_time, need_new_action, timer, timer_max, 2 spare
 *  [29 + 55nl + 4j ..] PD target of joint j in DeepMimic joint-frame convention (w,x,y,z or angle) */
int dm_get_snapshot(dm_handle* h, int env, double* h_out);
int dm_set_snapshot(dm_handle* h, int env, const double* h_in);
/* Whole-batch simulation state, for checkpoints and bit-exact resumption: every per-environment device block over the padded environments
 * (SIM, TIME, FLAGS with the reset counters, MANIFOLD, the AMP history, the task blocks, the active clips, the contact-load keys) and the host
 * state that changes later results (the expert draw counters, the mode, the current episode time limits), behind a header that names the
 * handle's configuration.  dm_state_size gives the blob's size in bytes; dm_save_state writes it to h_out and dm_load_state reads it from h_in
 * (host memory).  Both copy on the handle's stream and SYNCHRONISE it: they are meant for rare calls, off the per-step path.  dm_load_state
 * refuses a blob whose header differs from this handle (scene, environment counts, tile width, sizes, clip count, seed, global offset,
 * model) with a dm_last_error that names the field, and leaves the handle unchanged then.  A loaded handle continues exactly as the saved
 * one would have. */
int dm_state_size(dm_handle* h, size_t* bytes);
int dm_save_state(dm_handle* h, void* h_out);
int dm_load_state(dm_handle* h, const void* h_in);
/* profile build only (DM_PROFILE, `make -C deepmimic_b200/csrc profile`; fails in a normal build): per-warp cycle counters by code section of the
 * last dm_update's step kernel, 18 uint32 per warp, block-major ([num_blocks][warps_per_block][18], tools/section_profile.py names them).
 * h_out may be NULL to query the two sizes only. */
int dm_get_section_profile(dm_handle* h, uint32_t* h_out, int* num_blocks, int* warps_per_block);
int dm_get_counters(dm_handle* h, int64_t* h_out);           /* {kernel launches so far, row-capacity overflows seen (must stay 0)} */

#ifdef __cplusplus
}
#endif
#endif
