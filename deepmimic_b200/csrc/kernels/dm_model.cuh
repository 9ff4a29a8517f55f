// Flat, immutable device model ("model blob") and per-environment state layout for the batched
// DeepMimic step.  Everything the kernels need about a character / controller / clip is
// pre-digested on the host (capi.cu: build_device_model) from the reference's asset files:
//   multibody frames + inertias  <- cSimCharacter::BuildMultiBody   (R/DeepMimicCore/sim/SimCharacter.cpp:789-946)
//   exact-shape inertias for SPD <- cRBDUtil::BuildMomentInertia*   (R/DeepMimicCore/sim/RBDUtil.cpp:615-740)
//   PD gains / torque limits     <- cImpPDController::InitGains     (R/DeepMimicCore/sim/ImpPDController.cpp:97-127)
// All lengths are in Bullet's scaled units (x world_scale, sim/World.cpp:229-235), like the reference's
// physics world; observations / rewards divide back.
#pragma once
#include <cstdint>

#include "dm_math.cuh"

#include "dm_task.cuh"
#include "dm_task_ext.cuh"

namespace dmk {

constexpr int kMaxLinks = 32;   // one lane per link
constexpr int kMaxDofs = 96;    // 6 + joint dofs (humanoid3d 34, dog3d 70)
constexpr int kMaxChain = 24;   // longest root->leaf dof chain (humanoid3d 13, dog3d 22)
constexpr int kMaxChildren = 4;
constexpr int kStepMaxThreads = 448;    // dm_step_kernel: 28 (W=16) / 14 (W=32) environments per block (14 warps)
constexpr int kStepRegs = 128;          // registers per thread ptxas allocates for every dm_step_kernel instantiation (host-only launch plans; dm_create reads the real count)
constexpr int kManifoldFloats = 48;  // per link: 4 points x 12 floats
constexpr int kProfCounters = 16;    // DM_PROFILE builds: section cycle counters per warp of dm_step_kernel

enum DevJointType { kJRevolute = 0, kJSpherical = 1, kJFixed = 2 };
enum DevShape { kSBox = 1, kSCapsule = 2, kSSphere = 3 };

struct DevLink {
    int parent, jtype, ndof, dof0;        // dof0: index of first joint dof in the (6+ndofs) generalised vector
    int level, nchild, child[kMaxChildren];
    int depth0;                           // chain depth of the first joint dof (base dofs have depth 0..5)
    int last_depth;                       // deepest dof depth on the chain base -> this link (5 for links hanging off the base without dofs)
    int shape, fall_contact, end_eff, has_limit;
    uint32_t anc_mask;                    // bit a set <=> link a is an ancestor-or-self
    float mass;
    float inertiaB[3];                    // Bullet collision-shape inertia (diag, link frame)
    float inertiaD[3];                    // exact-shape inertia used by DeepMimic's SPD model
    float dvec[3], evec[3];               // joint pivot -> COM (this frame) ; parent COM -> pivot (parent frame)
    float zrot[4];                        // parent->this rotation at q = 0 (x,y,z,w)
    float axis[3];                        // revolute axis, this frame
    float kp, kd, tlim;                   // scaled units (x scale^2)
    float he[3];                          // box half extents / capsule (radius, halfHeight) / sphere (radius)
    float break_thr;
    float lim_lo, lim_hi;
    float child_rot[4];                   // DeepMimic joint frame -> body frame (x,y,z,w)  (cSimBodyJoint::mChildRot)
    float child_pos[3];                   // joint origin in the body frame, UNscaled (cSimBodyJoint::mChildPos)
    float joint_w;                        // normalised DiffWeight (SceneImitate.cpp:236-248)
    float att_pt[3], att_rot[4];          // DeepMimic joint attach point (parent joint frame, UNscaled) and attach rotation (x,y,z,w)
    float body_att[3];                    // body COM in its joint frame, UNscaled (BodyDefs.Attach*)
    int pose_off, pose_size;              // DeepMimic pose-vector slot of this joint
    int act_off, act_size;                // action-vector slot
};

struct DevModel {
    int nl, n, maxlevel, cs;              // links, 6+dofs, deepest tree level, chain stride
    int pose_dim, state_size, action_size, amp_obs_size, amp_local_root;
    int phase_input, rec_world_root_pos, rec_world_root_rot;
    int num_frames, loop_motion;
    int end_at_clip_end;                  // cSceneImitate::CheckTerminate only (SceneImitate.cpp:193-205): a finished non-looping clip fails the episode
    int enable_fall_end, enable_contact_fall, sync_root_pos, sync_root_rot, rand_rot_reset;
    float scale, gravity[3], friction;
    float total_mass;
    double motion_dur, cycle_period, query_dt, time_lim_min, time_lim_max, time_end_lim_max;
    float cycle_delta[3];
    // AMP task scenes (dm_task.cuh); task_kind == kTaskNone for imitate / imitate_amp
    int task_kind;
    TaskParams task;
    unsigned long long task_seed, env_id_base;   // draw stream: u01(task_seed, env_id_base + env, k)
    TaskExtParams taskx;                          // heading_amp_getup / strike_amp (dm_task_ext.cuh)
    int test_mode, pad_task_;                     // cRLScene::eMode, kept current by dm_set_mode in the task scenes
    DevLink link[kMaxLinks];
    uint8_t chain_dof[kMaxLinks][kMaxChain];  // dof index at chain depth d on the path base -> link (valid for d <= last depth of link)
    uint8_t dof_depth[kMaxDofs];
    uint8_t dof_link[kMaxDofs];           // owning link (base dofs: 0)
    // mocap tables live in separate device arrays: frame_times (double), frames / frame_vel (float, pose layout, root w-first quats)
};

// ---- clip dataset of --kin_ctrl clips (cClipsController, anim/ClipsController.cpp): the frames of all clips are concatenated in the
// mocap tables (clip 0 first, so a one-clip scene is laid out exactly like --kin_ctrl motion); one table per handle in global memory
constexpr int kMaxClips = 128;
struct ClipInfo {
    double dur;               // cMotion::GetDuration
    int frame_off;            // first frame of the clip in frame_times / frames / frame_vel (frame_times restart at 0 for every clip)
    int num_frames, loop;
    float cycle_delta[3];     // cKinController::CalcCycleRootDelta
    int is_getup;             // cSceneHeadingAMPGetup::mGetupMotionFlags
};
struct ClipTable {
    int num_clips, pad_;
    double cdf[kMaxClips];    // cClipsController::BuildClipsCDF
    ClipInfo info[kMaxClips];
};
// what the clip samplers read: DevModel (the scene's single clip) in the plain instantiations, this view of one dataset clip in the CLIPS ones
struct ClipModel {
    double motion_dur, query_dt;
    int loop_motion, num_frames, pose_dim;
    float cycle_delta[3];
};
__host__ __device__ inline ClipModel clip_model(const ClipInfo& c, int pose_dim, double query_dt) {
    ClipModel m; m.motion_dur = c.dur; m.query_dt = query_dt; m.loop_motion = c.loop; m.num_frames = c.num_frames; m.pose_dim = pose_dim;
    m.cycle_delta[0] = c.cycle_delta[0]; m.cycle_delta[1] = c.cycle_delta[1]; m.cycle_delta[2] = c.cycle_delta[2];
    return m;
}
// cClipsController::SelectNewMotion (ClipsController.cpp:226-236): std::upper_bound of a uniform draw in the CDF
__host__ __device__ inline int select_clip(const ClipTable& t, double u) {
    int lo = 0, hi = t.num_clips;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (t.cdf[mid] <= u) lo = mid + 1; else hi = mid; }
    return lo < t.num_clips ? lo : t.num_clips - 1;
}

// ---- per-environment state (env-major blocks; one tile of lanes reads a block with float4 loads)
// SIM block, floats:  [0..2] basePos [4..7] baseQuat(world->base) [8..10] baseOmega [12..14] baseVel
//                     [16 + 4 j ..] jointPos(j)  (spherical: quat xyzw; revolute: angle in .x)
//                     [16 + 4 nl + 4 j ..] jointVel(j) (xyz)
//                     [16 + 8 nl + 4 j ..] pdTarget(j) (body-frame quat xyzw / angle in .x)
__host__ __device__ inline int sim_stride(int nl) { return 16 + 12 * nl; }
// TIME block, doubles: kin_time, ctrl_time, init_time_offset, prev_action_time, timer_time, timer_max, origin[3], origin_rot[4] (w,x,y,z)
constexpr int kTimeDoubles = 16;
enum TimeSlot { kTKin = 0, kTCtrl = 1, kTInitOff = 2, kTPrevAct = 3, kTTimer = 4, kTTimerMax = 5, kTOrigin = 6, kTOriginRot = 9 };
// FLAG block, ints: need_new_action, done (sticky until reset), terminate, valid, fallen, overflow_rows
constexpr int kFlagInts = 8;
enum FlagSlot { kFNeedAction = 0, kFDone = 1, kFTerminate = 2, kFValid = 3, kFFallen = 4, kFRowOverflow = 5, kFUpdates = 6 };
// MANIFOLD block, floats: nl x 4 points x 12 = {valid, lAx,lAy,lAz, wBx,wBy,wBz, impN, impL1, impL2, dist, life}

struct DevState {
    float* sim;
    double* time;
    int* flags;
    float* manifold;
    float* hist;  // AMP history: DeepMimic pose | vel vectors (2 * pose_dim floats per env) of the simulated character at the last applied action
    unsigned int* prof;   // DM_PROFILE builds: kProfCounters per warp of every step-kernel block; null otherwise
    double* task; // AMP task scenes: kTaskDoubles per env (dm_task.cuh), null otherwise
    double* taskx; // ... and kTaskExtDoubles per env (dm_task_ext.cuh)
    int* clip;    // --kin_ctrl clips: active clip of every env, null for single-clip scenes
    const ClipTable* ctab;
    int num_envs;   // padded to a multiple of the step kernel's environments per block
    int num_real;   // environments the caller asked for; [num_real, num_envs) are padding: permanently "done", never reset, never simulated
};

// Output destinations of dm_observe_kernel: [0] is local, [1..n) the same slots of the peers' exchange buffers (NVLink P2P stores).
// obs: [num_envs x state_size], rew / done: [num_envs] floats; rew[0] / done[0] null = not wanted.
constexpr int kMaxFan = 8;
struct ObsFan {
    int n;
    float* obs[kMaxFan];
    float* rew[kMaxFan];
    float* done[kMaxFan];
};

// Row capacity of the constraint solver per tile width = row stride of the Y block.  W = 16 (humanoid3d): 2 rows per lane (8 foot points x 3 + limits
// <= 28).  W = 32: 52 = 16 points x 3 + 4 limit rows (dog3d: four feet flat + its four revolute joints at a limit), which is what lets 14
// dog environments share a block: on 148 SMs 2048 environments then run as ONE wave of 147 blocks instead of 171 blocks in two waves.  (The
// 132 SMs of an H100 would need two blocks of 8 per SM for one wave; DESIGN.md section 9 has what that lacks.)
__host__ __device__ constexpr int dm_step_y_stride(int W) { return W == 16 ? 32 : 52; }

// shared-memory layout of dm_step_kernel (float offsets inside one environment's block), filled by dm_step_layout on the host and
// passed by value as a kernel parameter (constant bank)
struct StepLayout {
    int nl, n, chain_len, maxrows, maxpts;
    int oU, oR, oA, oW, oV, oY, oLam, oRhs, oInv, oRl, oPp, oPi, oPr, oQ, oG, oZ;
    int env_floats, hot_floats;
};

}  // namespace dmk
