// C-ABI implementation (include/deepmimic_b200.h): host-side scene construction from the reference's asset
// formats, device model blob, launches of the sm_90a kernels.  No CPU fallback: every compute entry point
// launches CUDA work and fails loudly if the device / kernels are unavailable.
#include <cuda_runtime.h>

#include <algorithm>
#include <map>
#include <mutex>
#include <cmath>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <numeric>
#include <cstring>
#include <ctime>
#include <utility>
#include <memory>
#include <string>
#include <vector>

#include "../../include/deepmimic_b200.h"
#include "host/assets.hpp"
#include "kernels/dm_model.cuh"
#include "kernels/dm_pose_error.cuh"
#include "kernels/dm_render.cuh"

namespace dmk {
__global__ void dm_flags_kernel(DevState st, int32_t* out, int num_real_envs) {
    int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= num_real_envs) return;
    const int* f = st.flags + static_cast<size_t>(e) * kFlagInts;
    out[e * 4 + 0] = f[kFNeedAction]; out[e * 4 + 1] = f[kFDone]; out[e * 4 + 2] = f[kFTerminate]; out[e * 4 + 3] = f[kFValid];
}

// ---- multi-GPU exchange flags (dm_exchange_*): every rank owns one block {epoch[8], ack[8], status} that its peers write through P2P.
// epoch[r] = s + 1: rank r's rows of policy step s have arrived here; ack[r] = s + 1: rank r has finished reading the rows of step s there.
struct XchgFlags { unsigned long long epoch[8]; unsigned long long ack[8]; unsigned int status; unsigned int pad[31]; };
struct XchgPeers { int n; XchgFlags* f[8]; };
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// lane r publishes `value` into slot `me` of peer r's epoch (which = 0) or ack (which = 1) array.  The rows were stored by the preceding
// kernel of this stream; the system-scope fence + release store order them before the flag for the remote acquire load.
__global__ void dm_xchg_signal_kernel(XchgPeers P, int me, int which, unsigned long long value) {
    const int r = threadIdx.x;
    if (r >= P.n) return;
    __threadfence_system();
    st_release_sys(which == 0 ? &P.f[r]->epoch[me] : &P.f[r]->ack[me], value);
}
// lane r spins until this rank's own epoch[r] (which = 0) / ack[r] (which = 1) reaches `value`; gives up after `timeout_ns` and raises status
__global__ void dm_xchg_wait_kernel(XchgFlags* mine, int n, int which, unsigned long long value, unsigned long long timeout_ns) {
    const int r = threadIdx.x;
    if (r >= n) return;
    const unsigned long long* p = which == 0 ? &mine->epoch[r] : &mine->ack[r];
    unsigned long long t0;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    while (ld_acquire_sys(p) < value) {
        unsigned long long t1;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
        if (t1 - t0 > timeout_ns) { atomicOr(&mine->status, 1u << which); return; }
        __nanosleep(200);
    }
}
}  // namespace dmk

static thread_local std::string g_err;
// every compute entry point: refuse host-only handles (dm_load_host) loudly, then select the handle's device
#define DM_DEVICE(h)                                                                                                             \
    do {                                                                                                                         \
        if ((h)->stream == nullptr) { g_err = "host-only handle (dm_load_host): no device state, and there is no CPU fallback"; return fail(); } \
        DM_CUDA(cudaSetDevice((h)->device));                                                                                     \
    } while (0)
#define DM_CUDA(call)                                                                                         \
    do {                                                                                                      \
        cudaError_t e_ = (call);                                                                              \
        if (e_ != cudaSuccess) { g_err = std::string(#call) + ": " + cudaGetErrorString(e_); return fail(); } \
    } while (0)

struct dm_handle {
    dmh::SceneAssets sa;
    dmk::DevModel hm;        // host copy of the model blob
    dmk::DevModel* d_model = nullptr;
    dmk::DevState st{};
    double* d_frame_times = nullptr;
    float* d_frames = nullptr;
    float* d_frame_vel = nullptr;
    double* d_inj[3] = {nullptr, nullptr, nullptr};
    int32_t* d_flags4 = nullptr;
    float *d_amp = nullptr, *p_amp = nullptr;                              // staging for dm_amp_obs_host
    float *d_goal = nullptr, *p_goal = nullptr;                            // staging for dm_goal_host (task scenes)
    dmk::ClipTable ctab{};                                                  // host copy of the clip dataset table (task scenes)
    dmk::ClipTable* d_ctab = nullptr; int* d_clip_inj = nullptr;           // device table; injected clip ids (reset / expert observations)
    int total_frames = 0;
    float *d_act = nullptr, *d_obs = nullptr, *d_rew = nullptr;            // staging for dm_step_host
    float *p_act = nullptr, *p_obs = nullptr, *p_rew = nullptr; int32_t* p_flags = nullptr;  // pinned host staging
    cudaStream_t stream = nullptr;
    int device = 0, num_envs = 0, padded_envs = 0, W = 32, tiles = 2, maxrows = 36, smem_bytes = 0, mode = 0;
    dmk::DevPush* d_push = nullptr;   // push table (dm_set_pushes, dm_set_push_schedule): null until the first call, then the step launches use the push instantiations
    double* d_push_sched = nullptr;   // schedule block (dm_set_push_schedule): null on handles without a schedule; then d_push is the schedule's
    dmk::PushSchedule push_sched{};
    dmk::DevDyn* d_dyn = nullptr;       // dynamics table (dm_set_dynamics, dm_set_dynamics_randomization): null until the first call, then the step and
                                        // observation launches use the dynamics instantiations
    dmk::DevPush* d_push_none = nullptr;   // the dynamics step kernel's push table on a handle without pushes: every entry empty
    bool dyn_random = false;            // the table is drawn by dyn_rand at every reset (and owned by it)
    dmk::DynRand dyn_rand{};
    int* d_order = nullptr;   // placement of the environments in the step kernel's tiles (dm_set_env_order); st.order is it or null
    dmk::StepLayout lay{};
    uint64_t seed = 0, env_offset = 0;
    int64_t launches = 0;
    uint64_t amp_calls = 0;
    uint64_t expert_samples = 0;   // dm_sample_amp_obs_expert calls so far: the draw counter of its device stream
    std::vector<double> st_off, st_scale, act_off, act_scale, act_min, act_max, st_groups;
    // dm_step_host: page-locked-ness of the caller's buffers, looked up once per pointer (cudaPointerGetAttributes is a driver call)
    std::vector<std::pair<const void*, bool>> pin_cache;
    // dm_step_host_timing: phase events of the last dm_step_host call (created by dm_set_timing)
    // dm_exchange_*: one allocation {XchgFlags | 2 x [obs world*N*S | rew world*N | done world*N]}, mapped into the peers through CUDA IPC
    int x_rank = 0, x_world = 0;
    char* x_base = nullptr;                       // this rank's allocation
    char* x_peer[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};   // every rank's allocation as seen from here ([x_rank] = x_base)
    size_t x_data_off = 0, x_parity_bytes = 0;
    bool timing = false;
    cudaEvent_t tev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
    double host_ms[3] = {0, 0, 0};   // enqueue, wait (stream synchronize), staging copies
    std::vector<void*> dev_bufs, pinned_bufs;   // every buffer dm_create allocated (alloc_buffer), freed by dm_destroy
};

namespace {

int fail() { std::fprintf(stderr, "[deepmimic_b200] %s\n", g_err.c_str()); return 1; }

using dmh::Quat; using dmh::V3;
inline void put3(float* o, const V3& v, double s = 1.0) { o[0] = static_cast<float>(s * v.x); o[1] = static_cast<float>(s * v.y); o[2] = static_cast<float>(s * v.z); }
inline void putq(float* o, const Quat& q) { o[0] = static_cast<float>(q.x); o[1] = static_cast<float>(q.y); o[2] = static_cast<float>(q.z); o[3] = static_cast<float>(q.w); }

// Frame velocities of the clip, like cMotion::BuildFrameVel with cKinCharacter::CalcFrameVel -> cKinTree::CalcVel
// (R/DeepMimicCore/anim/Motion.cpp:170-191, anim/KinTree.cpp:1281-1316): world-frame rotation vector for the root,
// joint-local rotation vector for spherical joints, finite differences elsewhere.
std::vector<double> build_frame_vel(const dmh::CharModel& cm, const dmh::MotionClip& mc) {
    const int D = cm.pose_dim;
    std::vector<double> fv(static_cast<size_t>(mc.num_frames) * D, 0.0);
    for (int f = 0; f + 1 < mc.num_frames; ++f) {
        const double* a = mc.frame(f); const double* b = mc.frame(f + 1);
        const double dt = mc.frame_times[f + 1] - mc.frame_times[f];
        double* o = &fv[static_cast<size_t>(f) * D];
        for (int k = 0; k < 3; ++k) o[k] = (b[k] - a[k]) / dt;
        Quat q0(a[3], a[4], a[5], a[6]), q1(b[3], b[4], b[5], b[6]);
        V3 w = dmh::quat_to_rotvec(q1 * dmh::conj(q0));
        o[3] = w.x / dt; o[4] = w.y / dt; o[5] = w.z / dt; o[6] = 0;
        for (int j = 1; j < cm.num_joints(); ++j) {
            const auto& jd = cm.joints[j];
            const int p = jd.param_offset;
            if (jd.type == dmh::kSpherical) {
                Quat r0(a[p], a[p + 1], a[p + 2], a[p + 3]), r1(b[p], b[p + 1], b[p + 2], b[p + 3]);
                V3 wl = dmh::quat_to_rotvec(dmh::conj(r0) * r1);
                o[p] = wl.x / dt; o[p + 1] = wl.y / dt; o[p + 2] = wl.z / dt; o[p + 3] = 0;
            } else for (int k = 0; k < jd.param_size; ++k) o[p + k] = (b[p + k] - a[p + k]) / dt;
        }
    }
    if (mc.num_frames > 1) std::copy(fv.begin() + static_cast<size_t>(mc.num_frames - 2) * D, fv.begin() + static_cast<size_t>(mc.num_frames - 1) * D,
                                     fv.begin() + static_cast<size_t>(mc.num_frames - 1) * D);
    return fv;
}

// Digest the assets into the flat device model.  Frames follow cSimCharacter::BuildMultiBody
// (R/DeepMimicCore/sim/SimCharacter.cpp:789-946): every link frame sits at the body's COM with the body's orientation.
bool build_device_model(dm_handle& H) {
    const dmh::SceneAssets& sa = H.sa;
    const dmh::CharModel& cm = sa.character;
    dmk::DevModel& M = H.hm;
    std::memset(&M, 0, sizeof(M));
    const int nl = cm.num_joints();
    if (nl > dmk::kMaxLinks) { g_err = "character has more links than lanes (32)"; return false; }
    if (cm.joints[0].type != dmh::kNone) { g_err = "only floating-base characters (root joint type 'none') are supported"; return false; }
    const double sc = sa.cfg.world_scale;
    M.nl = nl; M.scale = static_cast<float>(sc);
    M.gravity[0] = static_cast<float>(sa.cfg.gravity.x * sc); M.gravity[1] = static_cast<float>(sa.cfg.gravity.y * sc); M.gravity[2] = static_cast<float>(sa.cfg.gravity.z * sc);
    M.friction = static_cast<float>(0.9 * 0.9);   // link 0.9 (sim/SimCharacter.cpp:26) x ground 0.9 (sim/Ground.cpp:17), Bullet multiplies them
    M.pose_dim = cm.pose_dim;
    M.phase_input = sa.ctrl.enable_phase_input; M.rec_world_root_pos = sa.ctrl.record_world_root_pos; M.rec_world_root_rot = sa.ctrl.record_world_root_rot;
    M.state_size = (M.phase_input ? 1 : 0) + 1 + nl * 9 + nl * 6;
    M.amp_local_root = sa.cfg.enable_amp_obs_local_root ? 1 : 0;
    {   // cSceneImitateAMP::GetAMPObsSize (SceneImitateAMP.cpp:75-84,214-258)
        int pose_sz = 1 + 6, nee = 0;
        for (int j = 0; j < nl; ++j) { const auto& jd = cm.joints[j]; if (jd.is_end_eff) ++nee; if (j > 0) pose_sz += (jd.type == dmh::kSpherical) ? 6 : jd.param_size; }
        M.amp_obs_size = 2 * (pose_sz + 3 * nee + 6 + (cm.pose_dim - cm.joints[0].param_size));
    }
    M.num_frames = sa.motion.num_frames; M.loop_motion = sa.motion.loop;
    M.end_at_clip_end = (!sa.motion.loop && sa.cfg.scene == "imitate") ? 1 : 0;   // cSceneImitateAMP::CheckTerminate skips the motion-over test (SceneImitateAMP.cpp:185-189)
    M.enable_fall_end = sa.cfg.enable_fall_end; M.enable_contact_fall = sa.cfg.enable_char_contact_fall; M.sync_root_pos = sa.cfg.sync_char_root_pos;
    M.sync_root_rot = sa.cfg.sync_char_root_rot; M.rand_rot_reset = sa.cfg.enable_rand_rot_reset;
    M.motion_dur = sa.motion.duration(); M.cycle_period = sa.motion.duration(); M.query_dt = 1.0 / sa.ctrl.query_rate;
    M.time_lim_min = sa.cfg.time_lim_min; M.time_lim_max = sa.cfg.time_lim_max; M.time_end_lim_max = sa.cfg.time_end_lim_max;
    M.total_mass = static_cast<float>(cm.total_mass());
    {   // AMP task scenes (dm_task.cuh)
        const dmh::SceneConfig& c = sa.cfg;
        M.task_kind = c.scene == "target_amp" ? dmk::kTaskTarget : c.scene == "heading_amp" ? dmk::kTaskHeading :
                      c.scene == "heading_amp_getup" ? dmk::kTaskHeadingGetup : c.scene == "strike_amp" ? dmk::kTaskStrike : dmk::kTaskNone;
        {   // heading_amp_getup / strike_amp (dm_task_ext.cuh)
            dmk::TaskExtParams& X = M.taskx;
            X.getup_time = 0.0;
            for (int id : c.getup_motion_ids) {
                if (id < 0 || id >= static_cast<int>(sa.clips.size())) { g_err = "--getup_motion_ids out of range"; return false; }
                X.getup_time = std::max(X.getup_time, sa.clips[id].duration());   // cSceneHeadingAMPGetup::CalcGetupTime (:262-287)
            }
            X.getup_height_root = c.getup_height_root; X.getup_height_head = c.getup_height_head; X.recover_episode_prob = c.recover_episode_prob;
            for (int k = 0; k < 3; ++k) { X.target_min[k] = c.target_min[k]; X.target_max[k] = c.target_max[k]; }
            X.target_radius = c.target_radius; X.hit_reset_time = c.target_hit_reset_time; X.tar_reward_scale = c.tar_reward_scale; X.hit_tar_speed = c.hit_tar_speed;
            X.init_hit_prob = c.init_hit_prob; X.tar_far_prob = c.tar_far_prob; X.tar_near_dist = c.tar_near_dist;
            X.head_id = c.head_id;
            if (X.head_id < 0 || X.head_id >= nl) { g_err = "--head_id out of range"; return false; }
            if (static_cast<int>(c.strike_bodies.size()) > dmk::kMaxTaskBodies || static_cast<int>(c.fail_tar_contact_bodies.size()) > dmk::kMaxTaskBodies) {
                g_err = "more than 4 --strike_bodies / --fail_tar_contact_bodies"; return false;
            }
            X.n_strike = static_cast<int>(c.strike_bodies.size()); X.n_fail = static_cast<int>(c.fail_tar_contact_bodies.size());
            for (int k = 0; k < dmk::kMaxTaskBodies; ++k) {
                X.strike_bodies[k] = k < X.n_strike ? c.strike_bodies[k] : 0; X.fail_bodies[k] = k < X.n_fail ? c.fail_tar_contact_bodies[k] : 0;
                if (X.strike_bodies[k] < 0 || X.strike_bodies[k] >= nl || X.fail_bodies[k] < 0 || X.fail_bodies[k] >= nl) { g_err = "strike / fail body id out of range"; return false; }
            }
            if (M.task_kind == dmk::kTaskStrike && X.n_strike == 0) { g_err = "strike_amp needs --strike_bodies"; return false; }
            if (M.task_kind == dmk::kTaskHeadingGetup && !(X.getup_time > 0.0)) { g_err = "heading_amp_getup needs --getup_motion_ids"; return false; }
        }
        dmk::TaskParams& T = M.task;
        T.timer_min = c.rand_target_time_min; T.timer_max = c.rand_target_time_max;
        T.max_target_dist = c.max_target_dist; T.target_succ_dist = c.target_succ_dist; T.tar_fail_dist = c.tar_fail_dist; T.pos_reward_scale = c.pos_reward_scale;
        T.max_heading_turn_rate = c.max_heading_turn_rate; T.sharp_turn_prob = c.sharp_turn_prob; T.speed_change_prob = c.speed_change_prob;
        T.tar_speed_min = c.tar_speed_min; T.tar_speed_max = c.tar_speed_max; T.vel_reward_scale = c.vel_reward_scale; T.tar_speed = c.tar_speed;
        T.enable_min_tar_vel = c.enable_min_tar_vel ? 1 : 0;
        M.task_seed = H.seed ^ 0x7461736b73ull;   // "tasks": a stream of its own next to the reset draws
        M.env_id_base = H.env_offset;
    }
    {
        const double* fb = sa.motion.frame(0); const double* fe = sa.motion.frame(sa.motion.num_frames - 1);
        M.cycle_delta[0] = static_cast<float>(fe[0] - fb[0]); M.cycle_delta[1] = 0.f; M.cycle_delta[2] = static_cast<float>(fe[2] - fb[2]);
    }
    double wsum = 0;
    for (const auto& j : cm.joints) wsum += std::fabs(j.diff_weight);
    int dof = 6, act_off = 0, maxlevel = 0, maxdepth = 5;
    std::vector<int> last_depth(nl, 5);
    for (int j = 0; j < nl; ++j) {
        const auto& jd = cm.joints[j]; const auto& bd = cm.bodies[j];
        dmk::DevLink& L = M.link[j];
        L.parent = jd.parent;
        const bool root = jd.parent < 0;
        if (root || jd.type == dmh::kFixed) { L.jtype = dmk::kJFixed; L.ndof = 0; }
        else if (jd.type == dmh::kRevolute) { L.jtype = dmk::kJRevolute; L.ndof = 1; }
        else if (jd.type == dmh::kSpherical) { L.jtype = dmk::kJSpherical; L.ndof = 3; }
        else { g_err = "unsupported joint type in character (planar / prismatic joints are outside the hot path)"; return false; }
        L.dof0 = dof; dof += L.ndof;
        L.level = root ? 0 : M.link[jd.parent].level + 1;
        maxlevel = std::max(maxlevel, L.level);
        L.nchild = 0;
        if (!root) {
            dmk::DevLink& P = M.link[jd.parent];
            if (P.nchild >= dmk::kMaxChildren) { g_err = "a link has more than 4 children"; return false; }
            P.child[P.nchild++] = j;
        }
        const int pd = root ? 5 : last_depth[jd.parent];
        L.depth0 = pd + 1;
        last_depth[j] = pd + L.ndof;
        L.last_depth = last_depth[j];
        maxdepth = std::max(maxdepth, last_depth[j]);
        if (last_depth[j] >= dmk::kMaxChain) { g_err = "dof chain too long"; return false; }
        if (root) for (int d = 0; d < 6; ++d) { M.chain_dof[j][d] = static_cast<uint8_t>(d); M.dof_depth[d] = static_cast<uint8_t>(d); M.dof_link[d] = 0; }
        else for (int d = 0; d <= pd; ++d) M.chain_dof[j][d] = M.chain_dof[jd.parent][d];
        for (int d = 0; d < L.ndof; ++d) { M.chain_dof[j][L.depth0 + d] = static_cast<uint8_t>(L.dof0 + d); M.dof_depth[L.dof0 + d] = static_cast<uint8_t>(L.depth0 + d); M.dof_link[L.dof0 + d] = static_cast<uint8_t>(j); }
        L.anc_mask = (root ? 0u : M.link[jd.parent].anc_mask) | (1u << j);
        // ---- frames
        Quat this_to_parent = dmh::euler_to_quat(jd.attach_theta), body_to_this = dmh::euler_to_quat(bd.attach_theta);
        Quat pb_to_parent; V3 pb_attach;
        if (!root) { pb_to_parent = dmh::euler_to_quat(cm.bodies[jd.parent].attach_theta); pb_attach = cm.bodies[jd.parent].attach_pt; }
        Quat parent_to_pb = dmh::conj(pb_to_parent);
        Quat body_to_pb = parent_to_pb * this_to_parent * body_to_this;
        putq(L.zrot, dmh::conj(body_to_pb));
        V3 e = dmh::rotate(parent_to_pb, jd.attach_pt) - dmh::rotate(parent_to_pb, pb_attach);
        V3 d = dmh::rotate(dmh::conj(body_to_this), bd.attach_pt);
        put3(L.evec, e, sc); put3(L.dvec, d, sc);
        put3(L.axis, dmh::rotate(dmh::conj(body_to_this), V3(0, 0, 1)));
        putq(L.child_rot, dmh::conj(body_to_this));
        put3(L.child_pos, -1.0 * dmh::rotate(dmh::conj(body_to_this), bd.attach_pt));
        put3(L.att_pt, jd.attach_pt); putq(L.att_rot, this_to_parent); put3(L.body_att, bd.attach_pt);
        // ---- mass properties at scaled size
        L.mass = static_cast<float>(bd.mass);
        const double m = bd.mass;
        if (bd.shape == dmh::kShapeBox) {
            L.shape = dmk::kSBox;
            const double hx = 0.5 * sc * bd.param[0], hy = 0.5 * sc * bd.param[1], hz = 0.5 * sc * bd.param[2];
            L.he[0] = static_cast<float>(hx); L.he[1] = static_cast<float>(hy); L.he[2] = static_cast<float>(hz);
            const double ix = m / 12.0 * (4 * hy * hy + 4 * hz * hz), iy = m / 12.0 * (4 * hx * hx + 4 * hz * hz), iz = m / 12.0 * (4 * hx * hx + 4 * hy * hy);
            L.inertiaB[0] = L.inertiaD[0] = static_cast<float>(ix); L.inertiaB[1] = L.inertiaD[1] = static_cast<float>(iy); L.inertiaB[2] = L.inertiaD[2] = static_cast<float>(iz);
            L.break_thr = static_cast<float>(0.02 * std::sqrt(hx * hx + hy * hy + hz * hz));
        } else if (bd.shape == dmh::kShapeCapsule) {
            L.shape = dmk::kSCapsule;
            const double r = 0.5 * sc * bd.param[0], hgt = sc * bd.param[1], hh = 0.5 * hgt;
            L.he[0] = static_cast<float>(r); L.he[1] = static_cast<float>(hh); L.he[2] = 0.f;
            // Bullet 2.88: inertia of the capsule's bounding box with CONVEX_DISTANCE_MARGIN (0.04, scaled units) added to every half extent
            // (btCapsuleShape::calculateLocalInertia)
            const double mg = 0.04, lx = 2 * (r + mg), ly = 2 * (r + hh + mg), lz = 2 * (r + mg), sm = m * 0.08333333;
            L.inertiaB[0] = static_cast<float>(sm * (ly * ly + lz * lz)); L.inertiaB[1] = static_cast<float>(sm * (lx * lx + lz * lz)); L.inertiaB[2] = static_cast<float>(sm * (lx * lx + ly * ly));
            // DeepMimic SPD model: exact capsule (cRBDUtil::BuildMomentInertiaCapsule, RBDUtil.cpp:667-694)
            const double c_vol = M_PI * r * r * hgt, hs_vol = M_PI * 2.0 / 3.0 * r * r * r, dens = m / (c_vol + 2 * hs_vol), cmass = c_vol * dens, hsm = hs_vol * dens;
            const double x = cmass * (0.25 * r * r + hgt * hgt / 12.0) + 2 * hsm * (0.4 * r * r + 0.375 * r * hgt + 0.25 * hgt * hgt), y = (0.5 * cmass + 0.8 * hsm) * r * r;
            L.inertiaD[0] = static_cast<float>(x); L.inertiaD[1] = static_cast<float>(y); L.inertiaD[2] = static_cast<float>(x);
            L.break_thr = static_cast<float>(0.02 * std::sqrt(2 * r * r + (r + hh) * (r + hh)));
        } else if (bd.shape == dmh::kShapeSphere) {
            L.shape = dmk::kSSphere;
            const double r = 0.5 * sc * bd.param[0];
            L.he[0] = static_cast<float>(r);
            const double i = 0.4 * m * r * r;
            for (int k = 0; k < 3; ++k) L.inertiaB[k] = L.inertiaD[k] = static_cast<float>(i);
            L.break_thr = static_cast<float>(0.02 * std::sqrt(3.0) * r);
        } else { g_err = "unsupported body shape (box / capsule / sphere only)"; return false; }
        L.fall_contact = bd.fall_contact; L.end_eff = jd.is_end_eff;
        L.kp = static_cast<float>(sc * sc * (root ? 0.0 : sa.ctrl.pd[j].kp)); L.kd = static_cast<float>(sc * sc * (root ? 0.0 : sa.ctrl.pd[j].kd));
        L.tlim = std::isfinite(jd.torque_lim) ? static_cast<float>(sc * sc * jd.torque_lim) : 3.0e38f;
        L.has_limit = (L.jtype == dmk::kJRevolute && jd.lim_low[0] <= jd.lim_high[1]) ? 1 : 0;   // sic: sim/SimCharacter.cpp:958
        L.lim_lo = static_cast<float>(jd.lim_low[0]); L.lim_hi = static_cast<float>(jd.lim_high[0]);
        L.joint_w = static_cast<float>(jd.diff_weight / wsum);
        L.pose_off = jd.param_offset; L.pose_size = jd.param_size;
        L.act_off = act_off; L.act_size = root ? 0 : (jd.type == dmh::kSpherical ? 3 : jd.param_size);
        act_off += L.act_size;
    }
    M.n = dof; M.maxlevel = maxlevel; M.action_size = act_off;
    M.cs = ((maxdepth + 1 + 7) / 8) * 8;
    if (M.n > dmk::kMaxDofs) { g_err = "too many dofs"; return false; }
    return true;
}

// static tables the agent reads once (cCtController / cCtCtrlUtil, SURVEY.md A.3, 8(c)(7))
void build_statics(dm_handle& H) {
    const auto& cm = H.sa.character; const auto& M = H.hm;
    H.st_off.assign(M.state_size, 0.0); H.st_scale.assign(M.state_size, 1.0); H.st_groups.assign(M.state_size, 0.0);
    if (M.phase_input) { H.st_off[0] = -0.5; H.st_scale[0] = 2.0; H.st_groups[0] = -1.0; }   // CtController.cpp:54-69,268-279,364-371
    H.act_off.assign(M.action_size, 0.0); H.act_scale.assign(M.action_size, 1.0); H.act_min.assign(M.action_size, 0.0); H.act_max.assign(M.action_size, 0.0);
    for (int j = 1; j < M.nl; ++j) {
        const auto& jd = cm.joints[j]; const auto& L = M.link[j];
        if (jd.type == dmh::kSpherical) {
            for (int k = 0; k < 3; ++k) { H.act_off[L.act_off + k] = 0; H.act_scale[L.act_off + k] = 2.0 / (2.0 * M_PI); H.act_min[L.act_off + k] = -2.0 * M_PI; H.act_max[L.act_off + k] = 2.0 * M_PI; }
        } else if (jd.type == dmh::kRevolute) {
            double lo = jd.lim_low[0], hi = jd.lim_high[0];
            if (!(hi >= lo)) { lo = -M_PI; hi = M_PI; }
            H.act_off[L.act_off] = -0.5 * (hi + lo); H.act_scale[L.act_off] = 0.5 / (hi - lo);
            const double mean = 0.5 * (hi + lo), delta = hi - lo;
            H.act_min[L.act_off] = mean - 2 * delta; H.act_max[L.act_off] = mean + 2 * delta;
        }
    }
}

bool task_scene(const dm_handle* h) { return h->hm.task_kind != dmk::kTaskNone; }
int goal_size(const dmk::DevModel& M) { return M.task_kind == dmk::kTaskNone ? 0 : (M.task_kind >= dmk::kTaskHeadingGetup ? 4 : 3); }
// row of the kernel tables (dm_model.cuh) for the handle's tile width, and grid of the kPolicyBlock-thread kernels
int tile_index(const dm_handle* h) { return h->W == 32 ? 1 : 0; }
int policy_grid(const dm_handle* h) { return h->padded_envs / (dmk::kPolicyBlock / h->W); }

// the tail of every launch
int launched(dm_handle* h) {
    DM_CUDA(cudaGetLastError());
    h->launches++;
    return 0;
}

int launch_step(dm_handle* h, double dt, int n_updates) {
    // AMP task scenes: the variant that also advances the task block; handles with a push table (dm_set_pushes): the push kernel, which applies it
    // handles with a dynamics table (dm_set_dynamics*): the dynamics kernel, which also applies the push table if there is one
    const void* kern = h->d_dyn ? reinterpret_cast<const void*>(dmk::kStepDynKernels[tile_index(h)][task_scene(h)])
                     : h->d_push ? reinterpret_cast<const void*>(dmk::kStepPushKernels[tile_index(h)][task_scene(h)])
                                 : reinterpret_cast<const void*>(dmk::kStepKernels[tile_index(h)][task_scene(h)]);
    // opt in to the large dynamic shared-memory carve-out; the limit is raised whenever a handle needs more than any earlier one on
    // this device (attributes are per device and per function: several handles of different sizes may live in one process)
    static std::mutex mu;
    static std::map<std::pair<int, const void*>, int> configured;   // (device, kernel) -> bytes configured
    {
        std::lock_guard<std::mutex> lock(mu);
        int& have = configured[{h->device, kern}];
        if (h->smem_bytes > have) {
            DM_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, h->smem_bytes));
            DM_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
            // the ordering kernel runs between two step launches: it gets the step kernel's carve-out
            DM_CUDA(cudaFuncSetAttribute(dmk::dm_env_order_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
            have = h->smem_bytes;
        }
    }
    if (h->st.order) {
        dmk::dm_env_order_kernel<<<1, dmk::kEnvOrderThreads, 0, h->stream>>>(h->st.load, h->padded_envs, h->tiles, h->W, h->d_order);
        if (launched(h)) return 1;
    }
    const dim3 grid(h->padded_envs / h->tiles), block(h->tiles * h->W);
    if (h->d_dyn)
        dmk::kStepDynKernels[tile_index(h)][task_scene(h)]<<<grid, block, h->smem_bytes, h->stream>>>(h->d_model, h->st, h->d_frame_times, h->d_frames, dt,
                                                                                                     n_updates, h->sa.cfg.num_sim_substeps, h->lay,
                                                                                                     h->d_push ? h->d_push : h->d_push_none, h->d_dyn);
    else if (h->d_push)
        dmk::kStepPushKernels[tile_index(h)][task_scene(h)]<<<grid, block, h->smem_bytes, h->stream>>>(h->d_model, h->st, h->d_frame_times, h->d_frames, dt,
                                                                                                      n_updates, h->sa.cfg.num_sim_substeps, h->lay, h->d_push);
    else
        dmk::kStepKernels[tile_index(h)][task_scene(h)]<<<grid, block, h->smem_bytes, h->stream>>>(h->d_model, h->st, h->d_frame_times, h->d_frames, dt, n_updates,
                                                                                                  h->sa.cfg.num_sim_substeps, h->lay);
    return launched(h);
}
int launch_observe_fan(dm_handle* h, const dmk::ObsFan& fan) {
    const size_t smem = static_cast<size_t>(dmk::kPolicyBlock / h->W) * h->hm.state_size * sizeof(float);   // the block's observation rows, staged for 16-byte stores
    if (h->d_dyn) {   // the reward's COM velocities with the environments' own masses
        const dmk::ObserveDynKernel kern = dmk::kObserveDynKernels[tile_index(h)][task_scene(h)];
        kern<<<policy_grid(h), dmk::kPolicyBlock, smem, h->stream>>>(h->d_model, h->st, h->d_frame_times, h->d_frames, h->d_frame_vel, fan, h->num_envs, h->d_dyn);
        return launched(h);
    }
    const dmk::ObserveKernel kern = dmk::kObserveKernels[tile_index(h)][task_scene(h)];   // task scenes: every environment's own active clip
    kern<<<policy_grid(h), dmk::kPolicyBlock, smem, h->stream>>>(h->d_model, h->st, h->d_frame_times, h->d_frames, h->d_frame_vel, fan, h->num_envs);
    return launched(h);
}
int launch_observe(dm_handle* h, float* d_state, float* d_reward) {
    dmk::ObsFan fan{};
    fan.n = 1; fan.obs[0] = d_state; fan.rew[0] = d_reward; fan.done[0] = nullptr;
    return launch_observe_fan(h, fan);
}
// clip: injected clip ids, task scenes only (dm_reset_clips refuses them elsewhere)
int launch_reset(dm_handle* h, int force, const double* kt, const double* mt, const double* th, const int* clip) {
    // task scenes: per-environment clip of the dataset, action history kept across resets
    const dmk::ResetKernel kern = dmk::kResetKernels[tile_index(h)][task_scene(h)];
    kern<<<policy_grid(h), dmk::kPolicyBlock, 0, h->stream>>>(h->d_model, h->st, h->d_frame_times, h->d_frames, h->d_frame_vel, force, kt, mt, th, h->seed,
                                                              h->env_offset, h->mode, clip);
    return launched(h);
}
// d_clips: expert samples from per-environment dataset clips (task scenes), null otherwise
int launch_amp(dm_handle* h, float* d_out, int expert, const double* d_times, const int* d_clips) {
    const dmk::AmpObsKernel kern = dmk::kAmpObsKernels[tile_index(h)][d_clips != nullptr];
    kern<<<policy_grid(h), dmk::kPolicyBlock, 0, h->stream>>>(h->d_model, h->st, h->d_frame_times, h->d_frames, h->d_frame_vel, d_out, expert, d_times,
                                                              h->num_envs, d_clips);
    return launched(h);
}
// pose / vel: [num_envs x pose_dim] rows of the real environments, either may be null
int launch_pose(dm_handle* h, float* d_pose, float* d_vel) {
    const int E = dmk::kPoseEnvsPerBlock;
    const size_t smem = static_cast<size_t>(E) * 2 * h->hm.pose_dim * sizeof(float);
    dmk::dm_pose_kernel<<<(h->num_envs + E - 1) / E, E * h->hm.nl, smem, h->stream>>>(h->d_model, h->st, d_pose, d_vel, h->num_envs);
    return launched(h);
}

// Copies bytes [off, off + bytes) of the host model blob into the device one, stream-ordered; host-only handles have no device blob.
int upload_model(dm_handle* h, size_t off, size_t bytes) {
    if (h->stream == nullptr) return 0;
    DM_CUDA(cudaSetDevice(h->device));
    DM_CUDA(cudaMemcpyAsync(reinterpret_cast<char*>(h->d_model) + off, reinterpret_cast<const char*>(&h->hm) + off, bytes, cudaMemcpyHostToDevice, h->stream));
    DM_CUDA(cudaStreamSynchronize(h->stream));
    return 0;
}
static_assert(offsetof(dmk::DevModel, time_lim_max) == offsetof(dmk::DevModel, time_lim_min) + sizeof(double), "time limits must be adjacent");
int upload_time_limits(dm_handle* h) { return upload_model(h, offsetof(dmk::DevModel, time_lim_min), 2 * sizeof(double)); }

// Copies one value per real environment into a device array of padded_envs entries.  The padding rows repeat the last real environment;
// no kernel reads them.  Waits for the copy: the staging vector is pageable.
template <class T>
int stage_envs(dm_handle* h, const T* src, T* dst) {
    std::vector<T> tmp(h->padded_envs);
    for (int e = 0; e < h->padded_envs; ++e) tmp[e] = src[std::min(e, h->num_envs - 1)];
    DM_CUDA(cudaMemcpyAsync(dst, tmp.data(), sizeof(T) * tmp.size(), cudaMemcpyHostToDevice, h->stream));
    DM_CUDA(cudaStreamSynchronize(h->stream));
    return 0;
}

// A buffer of `count` T that the handle owns until dm_destroy: on the device (kZeroed: cleared there) or page-locked on the host.
enum BufferKind { kDevice, kZeroed, kPinned };
template <class T>
int alloc_buffer(dm_handle* h, T** p, size_t count, BufferKind kind = kDevice) {
    if (kind == kPinned) {
        DM_CUDA(cudaMallocHost(p, count * sizeof(T)));
        h->pinned_bufs.push_back(*p);
        return 0;
    }
    DM_CUDA(cudaMalloc(p, count * sizeof(T)));
    h->dev_bufs.push_back(*p);
    if (kind == kZeroed) DM_CUDA(cudaMemset(*p, 0, count * sizeof(T)));
    return 0;
}

// Offsets of the SIM block (dm_model.cuh, floats) and of the snapshot (include/deepmimic_b200.h, doubles) of an nl-link character, after their
// fixed base-body part
struct SimOffsets {
    int jpos = 16, jvel, pd;
    explicit SimOffsets(int nl) : jvel(16 + 4 * nl), pd(16 + 8 * nl) {}
};
struct SnapshotOffsets {
    int jpos = 13, jvel, manifold, clocks, pd, size;
    explicit SnapshotOffsets(int nl) : jvel(13 + 4 * nl), manifold(13 + 7 * nl), clocks(13 + 55 * nl), pd(29 + 55 * nl), size(29 + 59 * nl) {}
};

}  // namespace

// Launch plan of dm_step_kernel: tile width, row capacity, shared-memory layout, environments per block, padded environment count.  Shared
// memory and kStepMaxThreads cap the environments per block; the environments are spread evenly over the fewest waves of blocks that hold them,
// since a wave takes as long as its fullest block.  A wave is one block per SM, or two when two blocks of the even split fit an SM's shared
// memory (smem_sm, with reserved bytes per block) and its register file (regs per thread): the kernel is latency-bound, so two blocks of 16
// humanoid environments per SM run in one wave what one block per SM needs two waves for.  With equally many waves the larger blocks win.  Pure
// host arithmetic (also reachable without a device through dm_plan_launch, for the CPU tests of the wave property).
static bool plan_launch(dm_handle& H, int num_envs, int smem_optin, int sms, int smem_sm, int smem_reserved, int regs) {
    const auto& M = H.hm;
    H.W = (M.nl <= 16) ? 16 : 32;   // lanes per environment: one lane per link
    H.maxrows = dmk::dm_step_y_stride(H.W);   // humanoid3d: 8 foot points x 3 + limit rows <= 28 of 32; dog3d: 4 feet x 4 points x 3 + 4 limit rows = 52
    int chain_len = 0;
    for (int j = 0; j < M.nl; ++j) chain_len = std::max(chain_len, M.link[j].last_depth + 1);
    dmk::dm_step_layout(M.nl, M.n, chain_len, H.maxrows, H.W, &H.lay);
    const int per_env = H.lay.env_floats * 4;
    const int hot = H.lay.hot_floats * 4 + 1024;
    const int max_tiles = std::min(dmk::kStepMaxThreads / H.W, (smem_optin - hot) / per_env);
    const int min_tiles = (H.W == 16) ? 2 : 1;   // W = 16: two environments share a warp
    if (max_tiles < min_tiles) {
        g_err = "not enough shared memory per block for one environment tile (need " + std::to_string(hot + min_tiles * per_env) + " bytes, the device offers " +
                std::to_string(static_cast<long long>(smem_optin)) + ")";
        return false;
    }
    auto even_split = [&](int slots, int cap) {   // environments per block when num_envs is spread evenly over waves of `slots` blocks
        const int waves = ((num_envs + cap - 1) / cap + slots - 1) / slots;
        int t = std::min(cap, std::max(min_tiles, (num_envs + waves * slots - 1) / (waves * slots)));
        if (H.W == 16 && (t & 1)) t = (t + 1 <= cap) ? t + 1 : t - 1;   // whole warps; t >= 2 here, so t - 1 >= 2 when odd
        return std::make_pair(waves, t);
    };
    auto [waves, tiles] = even_split(sms, max_tiles);
    {   // two blocks per SM: each within half the SM's shared memory and registers
        const int cap2 = std::min({max_tiles, (smem_sm / 2 - smem_reserved - hot) / per_env, 65536 / (2 * regs * H.W)});
        if (cap2 >= min_tiles) {
            const auto [waves2, tiles2] = even_split(2 * sms, cap2);
            if (waves2 < waves) { waves = waves2; tiles = tiles2; }
        }
    }
    H.tiles = tiles;
    const int quantum = (tiles * (64 / H.W)) / std::__gcd(tiles, 64 / H.W);   // multiple of both the update block and the 64-thread policy blocks
    H.padded_envs = ((num_envs + quantum - 1) / quantum) * quantum;
    H.smem_bytes = dmk::dm_step_smem_bytes(H.lay, H.tiles) + 1024;
    return true;
}

extern "C" {

const char* dm_last_error(void) { return g_err.c_str(); }
void dm_set_last_error(const char* msg) { g_err = msg ? msg : ""; }   // other translation units of the library (mlp_capi.cu) report through the same string

// host half of dm_create: argument / asset loading and the flat model (no device work)
static bool load_host_model(dm_handle& H, const char* asset_root, int argc, const char** argv) {
    try {
        std::vector<std::string> args(argv, argv + argc);
        dmh::ArgParser ap;
        ap.LoadArgs(args);
        std::string root = asset_root ? asset_root : "", arg_file;
        if (ap.ParseString("arg_file", arg_file) && !ap.LoadFile(dmh::resolve_path(root, arg_file))) throw std::runtime_error("Failed to load args from: " + arg_file);
        std::string timer_type;
        if (ap.ParseString("timer_type", timer_type) && timer_type != "" && timer_type != "uniform")   // cTimer::ParseTypeStr (util/Timer.cpp:26-43)
            throw std::runtime_error("Unsupported timer type " + timer_type + " (supported: uniform)");
        H.sa = dmh::load_scene_assets(ap, root);
        // scenes on the accelerated path: "imitate" and its AMP variant (same character, controller, clip and dynamics; AMP observations on top).
        // The AMP task scenes (heading / target / dribble / strike) add goals, task rewards and clip datasets that are not built: refuse them loudly.
        // options of the reference's scene that the batched path does not implement are refused, never ignored
        {
            const dmh::SceneConfig& c = H.sa.cfg;
            std::vector<std::string> v;
            if (!c.char_ctrl.empty() && c.char_ctrl != "ct_pd") throw std::runtime_error("Unsupported character controller: " + c.char_ctrl + " (supported: ct_pd)");
            if (ap.ParseStrings("character_files", v) && v.size() > 1) throw std::runtime_error("Unsupported: more than one character per scene");
            if (ap.ParseStrings("char_types", v) && !v.empty() && v[0] != "general") throw std::runtime_error("Unsupported character type: " + v[0] + " (supported: general)");
            bool soft = false;
            if (ap.ParseBool("enable_char_soft_contact", soft) && soft) throw std::runtime_error("Unsupported: --enable_char_soft_contact true");
            if (c.enable_root_rot_fail) throw std::runtime_error("Unsupported: --enable_root_rot_fail true");
            if (c.is_task_scene() && c.sync_char_root_rot) throw std::runtime_error("Unsupported: --sync_char_root_rot true in an AMP task scene");
            if (!c.terrain_file.empty()) {   // cGroundBuilder: only the flat plane (data/terrain/plane.txt) is on the path
                dmh::Json t = dmh::Json::parseFile(dmh::resolve_path(root, c.terrain_file));
                if (t["Type"].asString("") != "plane") throw std::runtime_error("Unsupported terrain type: " + t["Type"].asString("") + " (supported: plane)");
            }
        }
        // Scenes on the accelerated path: imitate, imitate_amp, and the AMP task scenes target_amp / heading_amp / heading_amp_getup /
        // strike_amp (goals, task rewards, clip datasets; checked against the oracle on the GPU: tests/test_task_scenes_gpu.py,
        // tests/test_task_ext_gpu.py).  Every other scene name is refused.
        const bool task_scene = H.sa.cfg.is_task_scene();   // target_amp, heading_amp, heading_amp_getup, strike_amp
        const std::string& scn = H.sa.cfg.scene;
        if (!task_scene && scn != "imitate" && scn != "imitate_amp")
            throw std::runtime_error("Unsupported scene: " + scn + " (supported: imitate, imitate_amp, target_amp, heading_amp, heading_amp_getup, strike_amp)");
        if (H.sa.clips.size() != 1 && !task_scene)
            throw std::runtime_error("Unsupported kinematic controller: clips with more than one clip outside the AMP task scenes (supported: motion)");
        if (static_cast<int>(H.sa.clips.size()) > dmk::kMaxClips) throw std::runtime_error("clip dataset larger than the device clip table (" + std::to_string(dmk::kMaxClips) + ")");
    } catch (const std::exception& e) { g_err = e.what(); return false; }
    if (!build_device_model(H)) return false;
    build_statics(H);
    return true;
}

dm_handle* dm_load_host(const char* asset_root, int argc, const char** argv) {
    std::unique_ptr<dm_handle> h(new dm_handle());
    if (!load_host_model(*h, asset_root, argc, argv)) { fail(); return nullptr; }
    return h.release();
}

int dm_plan_launch(dm_handle* h, int num_envs, int smem_bytes_per_block, int num_sms, int* out) {
    if (!h || num_envs <= 0 || num_sms <= 0) { g_err = "dm_plan_launch: bad arguments"; return fail(); }
    dm_handle tmp;
    tmp.hm = h->hm;
    // an SM holds the per-block maximum plus the 1 KB the runtime reserves per block (H100: 227 KB + 1 KB = 228 KB)
    if (!plan_launch(tmp, num_envs, smem_bytes_per_block, num_sms, smem_bytes_per_block + 1024, 1024, dmk::kStepRegs)) return fail();
    out[0] = tmp.W; out[1] = tmp.tiles; out[2] = tmp.padded_envs / tmp.tiles; out[3] = tmp.smem_bytes; out[4] = tmp.maxrows; out[5] = tmp.lay.env_floats;
    out[6] = tmp.lay.hot_floats; out[7] = tmp.lay.oY; out[8] = tmp.padded_envs;
    return 0;
}

int dm_get_model_info(dm_handle* h, int kind, int* out) {
    const auto& M = h->hm;
    switch (kind) {
        case DM_INFO_PARENTS: for (int j = 0; j < M.nl; ++j) out[j] = M.link[j].parent; break;
        case DM_INFO_JOINT_TYPES: for (int j = 0; j < M.nl; ++j) out[j] = M.link[j].jtype; break;
        case DM_INFO_DOF_OFFSETS: for (int j = 0; j < M.nl; ++j) out[j] = M.link[j].dof0; break;
        case DM_INFO_POSE_OFFSETS: for (int j = 0; j < M.nl; ++j) out[j] = M.link[j].pose_off; break;
        case DM_INFO_FALL_BODIES: for (int j = 0; j < M.nl; ++j) out[j] = M.link[j].fall_contact; break;
        case DM_INFO_END_EFFECTORS: for (int j = 0; j < M.nl; ++j) out[j] = M.link[j].end_eff; break;
        case DM_INFO_LAYOUT: out[0] = M.nl; out[1] = M.n; out[2] = M.cs; out[3] = M.maxlevel; out[4] = M.num_frames; out[5] = M.loop_motion; break;
        default: g_err = "dm_get_model_info: bad kind"; return fail();
    }
    return 0;
}

// Per-link model constants as the kernels use them (24 doubles per link): mass, Bullet inertia[3], DeepMimic inertia[3], dvec[3], evec[3],
// zrot (x,y,z,w), axis[3], half extents[3], breaking threshold.  Scaled units.  For the independent known-answer tests of the loader.
int dm_get_link_table(dm_handle* h, double* out) {
    const auto& M = h->hm;
    for (int j = 0; j < M.nl; ++j) {
        const dmk::DevLink& L = M.link[j];
        double* o = out + 24 * j;
        o[0] = L.mass;
        for (int k = 0; k < 3; ++k) { o[1 + k] = L.inertiaB[k]; o[4 + k] = L.inertiaD[k]; o[7 + k] = L.dvec[k]; o[10 + k] = L.evec[k]; o[17 + k] = L.axis[k]; o[20 + k] = L.he[k]; }
        for (int k = 0; k < 4; ++k) o[13 + k] = L.zrot[k];
        o[23] = L.break_thr;
    }
    return 0;
}

// device half of dm_create: launch plan, buffers, mocap tables and the initial state (the caller destroys the handle when it fails)
static int create_device_state(dm_handle* h, int num_envs, int device) {
    DM_CUDA(cudaSetDevice(device));
    h->device = device;
    const auto& M = h->hm;
    {
        cudaDeviceProp prop;
        DM_CUDA(cudaGetDeviceProperties(&prop, device));
        int regs = 0;   // registers per thread of the step kernel: the most any instantiation was compiled with
        for (const auto& row : dmk::kStepKernels) for (const dmk::StepKernel f : row) {
            cudaFuncAttributes fa;
            DM_CUDA(cudaFuncGetAttributes(&fa, f));
            regs = std::max(regs, fa.numRegs);
        }
        if (!plan_launch(*h, num_envs, static_cast<int>(prop.sharedMemPerBlockOptin), prop.multiProcessorCount, static_cast<int>(prop.sharedMemPerMultiprocessor),
                         static_cast<int>(prop.reservedSharedMemPerBlock), regs)) return fail();
    }
    const size_t N = static_cast<size_t>(h->padded_envs);
    const int ss = dmk::sim_stride(M.nl);
    // mocap tables: the frames of every clip of the scene, concatenated (one clip unless --kin_ctrl clips; clip 0 = the model's clip)
    h->total_frames = 0;
    h->ctab = dmk::ClipTable{};
    h->ctab.num_clips = static_cast<int>(h->sa.clips.size());
    for (size_t c = 0; c < h->sa.clips.size(); ++c) {
        const dmh::MotionClip& mc = h->sa.clips[c];
        dmk::ClipInfo& ci = h->ctab.info[c];
        ci.dur = mc.duration(); ci.frame_off = h->total_frames; ci.num_frames = mc.num_frames; ci.loop = mc.loop ? 1 : 0;
        const double* fb = mc.frame(0); const double* fe = mc.frame(mc.num_frames - 1);
        ci.cycle_delta[0] = static_cast<float>(fe[0] - fb[0]); ci.cycle_delta[1] = 0.f; ci.cycle_delta[2] = static_cast<float>(fe[2] - fb[2]);
        h->ctab.cdf[c] = h->sa.clip_cdf[c];
        ci.is_getup = std::find(h->sa.cfg.getup_motion_ids.begin(), h->sa.cfg.getup_motion_ids.end(), static_cast<int>(c)) != h->sa.cfg.getup_motion_ids.end() ? 1 : 0;
        h->total_frames += mc.num_frames;
    }
    const size_t TF = static_cast<size_t>(h->total_frames);
    DM_CUDA(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    if (alloc_buffer(h, &h->d_model, 1) || alloc_buffer(h, &h->st.sim, N * ss) || alloc_buffer(h, &h->st.time, N * dmk::kTimeDoubles, kZeroed) ||
        alloc_buffer(h, &h->st.flags, N * dmk::kFlagInts, kZeroed) || alloc_buffer(h, &h->st.manifold, N * M.nl * dmk::kManifoldFloats, kZeroed) ||
        alloc_buffer(h, &h->d_frame_times, TF) || alloc_buffer(h, &h->d_frames, TF * M.pose_dim) || alloc_buffer(h, &h->d_frame_vel, TF * M.pose_dim) ||
        alloc_buffer(h, &h->d_flags4, N * 4) || alloc_buffer(h, &h->d_amp, N * M.amp_obs_size) || alloc_buffer(h, &h->p_amp, N * M.amp_obs_size, kPinned) ||
        alloc_buffer(h, &h->st.hist, N * 2 * M.pose_dim) || alloc_buffer(h, &h->d_act, N * std::max(1, M.action_size)) ||
        alloc_buffer(h, &h->d_obs, N * M.state_size) || alloc_buffer(h, &h->d_rew, N) || alloc_buffer(h, &h->p_act, N * std::max(1, M.action_size), kPinned) ||
        alloc_buffer(h, &h->p_obs, N * M.state_size, kPinned) || alloc_buffer(h, &h->p_rew, N, kPinned) || alloc_buffer(h, &h->p_flags, N * 4, kPinned))
        return 1;
    for (auto& p : h->d_inj) if (alloc_buffer(h, &p, N)) return 1;
    if (alloc_buffer(h, &h->st.load, N) || alloc_buffer(h, &h->d_order, N)) return 1;
    {   // no contact load known yet; the padding environments sort last
        std::vector<int> load(N, 0), ident(N);
        std::fill(load.begin() + h->num_envs, load.end(), dmk::kLoadPadding);
        std::iota(ident.begin(), ident.end(), 0);
        DM_CUDA(cudaMemcpy(h->st.load, load.data(), N * sizeof(int), cudaMemcpyHostToDevice));
        DM_CUDA(cudaMemcpy(h->d_order, ident.data(), N * sizeof(int), cudaMemcpyHostToDevice));
    }
    h->st.order = (h->W == 16) ? h->d_order : nullptr;   // dm_set_env_order: W = 32 handles keep index placement
#ifdef DM_PROFILE
    // blocks x warps per block
    if (alloc_buffer(h, &h->st.prof, static_cast<size_t>(h->padded_envs / h->tiles) * (h->tiles * h->W / 32) * dmk::kProfCounters, kZeroed)) return 1;
#endif
    h->st.num_envs = h->padded_envs; h->st.num_real = h->num_envs;
    if (task_scene(h)) {
        if (alloc_buffer(h, &h->st.task, N * dmk::kTaskDoubles, kZeroed) || alloc_buffer(h, &h->st.taskx, N * dmk::kTaskExtDoubles, kZeroed) ||
            alloc_buffer(h, &h->d_goal, N * 4) || alloc_buffer(h, &h->p_goal, N * 4, kPinned) || alloc_buffer(h, &h->st.clip, N, kZeroed) ||
            alloc_buffer(h, &h->d_clip_inj, N) || alloc_buffer(h, &h->d_ctab, 1))
            return 1;
        DM_CUDA(cudaMemcpy(h->d_ctab, &h->ctab, sizeof(dmk::ClipTable), cudaMemcpyHostToDevice));
    }
    h->st.ctab = h->d_ctab;
    std::vector<float> frames(TF * M.pose_dim), fvel(frames.size());
    std::vector<double> ftimes(TF);
    for (size_t c = 0; c < h->sa.clips.size(); ++c) {
        const dmh::MotionClip& mc = h->sa.clips[c];
        const std::vector<double> fv = build_frame_vel(h->sa.character, mc);
        const size_t off = static_cast<size_t>(h->ctab.info[c].frame_off);
        std::copy(mc.frame_times.begin(), mc.frame_times.end(), ftimes.begin() + off);
        for (size_t i = 0; i < mc.frames.size(); ++i) { frames[off * M.pose_dim + i] = static_cast<float>(mc.frames[i]); fvel[off * M.pose_dim + i] = static_cast<float>(fv[i]); }
    }
    DM_CUDA(cudaMemcpy(h->d_model, &h->hm, sizeof(dmk::DevModel), cudaMemcpyHostToDevice));
    DM_CUDA(cudaMemcpy(h->d_frame_times, ftimes.data(), sizeof(double) * TF, cudaMemcpyHostToDevice));
    DM_CUDA(cudaMemcpy(h->d_frames, frames.data(), sizeof(float) * frames.size(), cudaMemcpyHostToDevice));
    DM_CUDA(cudaMemcpy(h->d_frame_vel, fvel.data(), sizeof(float) * fvel.size(), cudaMemcpyHostToDevice));
    if (h->padded_envs > h->num_envs) {
        // padding environments (the step kernel works on whole blocks): marked done once and for all, so that every kernel skips them.  Left
        // alive they would stand on both feet without ever receiving an action -- 26 constraint rows each, the slowest block of the launch
        // (found with tools/section_profile.py in round 2: the last block set the kernel time).
        std::vector<int> fl(static_cast<size_t>(h->padded_envs - h->num_envs) * dmk::kFlagInts, 0);
        for (int e = 0; e < h->padded_envs - h->num_envs; ++e) { fl[static_cast<size_t>(e) * dmk::kFlagInts + dmk::kFDone] = 1; fl[static_cast<size_t>(e) * dmk::kFlagInts + dmk::kFValid] = 1; }
        DM_CUDA(cudaMemcpy(h->st.flags + static_cast<size_t>(h->num_envs) * dmk::kFlagInts, fl.data(), fl.size() * sizeof(int), cudaMemcpyHostToDevice));
    }
    // the whole SIM block: zero but for the initial PD targets, identity / TargetTheta0 (cPDController::Init, PDController.cpp:99-112)
    std::vector<float> sim(N * ss, 0.f);
    const SimOffsets so(M.nl);
    for (size_t e = 0; e < N; ++e) for (int j = 0; j < M.nl; ++j) {
        float* t = &sim[e * ss + so.pd + 4 * j];
        if (M.link[j].jtype == dmk::kJSpherical) { t[0] = t[1] = t[2] = 0.f; t[3] = 1.f; }
        else t[0] = static_cast<float>(h->sa.ctrl.pd[j].target_theta[0]);
    }
    DM_CUDA(cudaMemcpy(h->st.sim, sim.data(), sim.size() * sizeof(float), cudaMemcpyHostToDevice));
    // the AMP history of every environment: the identity pose at rest (cSceneImitateAMP's mPrevPose / mPrevVel before any action, which the task
    // scenes keep across resets); the reset kernel overwrites it only in the non-task scenes (InitHist)
    std::vector<float> hist(N * 2 * M.pose_dim, 0.f);
    for (size_t e = 0; e < N; ++e) {
        float* p = &hist[e * 2 * M.pose_dim];
        p[3] = 1.f;
        for (int j = 1; j < M.nl; ++j) if (M.link[j].jtype == dmk::kJSpherical) p[M.link[j].pose_off] = 1.f;
    }
    DM_CUDA(cudaMemcpy(h->st.hist, hist.data(), hist.size() * sizeof(float), cudaMemcpyHostToDevice));
    return 0;
}

dm_handle* dm_create(const char* asset_root, int argc, const char** argv, int num_envs, int device, uint64_t seed, uint64_t global_env_offset) {
    std::unique_ptr<dm_handle> h(new dm_handle());
    if (!load_host_model(*h, asset_root, argc, argv)) { fail(); return nullptr; }
    if (num_envs <= 0) { g_err = "num_envs must be positive"; fail(); return nullptr; }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { g_err = "no CUDA device available: deepmimic_b200 has no CPU fallback"; fail(); return nullptr; }
    h->seed = seed; h->env_offset = global_env_offset; h->num_envs = num_envs;
    h->hm.task_seed = seed ^ 0x7461736b73ull; h->hm.env_id_base = global_env_offset;   // the model blob is uploaded by create_device_state
    if (create_device_state(h.get(), num_envs, device) != 0 || dm_reset(h.get(), 1, nullptr, nullptr, nullptr) != 0 || dm_sync(h.get()) != 0) {
        dm_destroy(h.release());
        return nullptr;
    }
    return h.release();
}

int dm_exchange_destroy(dm_handle* h);
void dm_destroy(dm_handle* h) {
    if (!h) return;
    cudaSetDevice(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    dm_exchange_destroy(h);
    for (void* p : h->dev_bufs) cudaFree(p);
    for (void* p : h->pinned_bufs) cudaFreeHost(p);
    for (auto& e : h->tev) if (e) cudaEventDestroy(e);
    if (h->stream) cudaStreamDestroy(h->stream);
    delete h;
}

int dm_get_dims(dm_handle* h, dm_dims* o) {
    const auto& M = h->hm;
    o->num_envs = h->num_envs; o->num_joints = M.nl; o->pose_dim = M.pose_dim; o->num_dofs = M.n; o->state_size = M.state_size; o->goal_size = goal_size(M); o->amp_obs_size = M.amp_obs_size;
    o->action_size = M.action_size; o->snapshot_size = SnapshotOffsets(M.nl).size;
    o->num_update_substeps = h->sa.cfg.num_update_substeps;
    o->updates_per_action = 20;
    o->motion_duration = M.motion_dur;
    return 0;
}
// cScene::GetName of the configured scene (SceneImitate.cpp:209, SceneImitateAMP.cpp:211, SceneTargetAMP.cpp:233, SceneHeadingAMP.cpp:153, ...)
int dm_get_scene_name(dm_handle* h, char* out, int cap) {
    const std::string& sc = h->sa.cfg.scene;
    const char* name = sc == "imitate_amp" ? "Imitate AMP" : sc == "target_amp" ? "Target AMP" : sc == "heading_amp" ? "Heading AMP" :
                       sc == "heading_amp_getup" ? "Heading AMP Getup" : sc == "strike_amp" ? "Strike AMP" : "Imitate";
    if (cap <= 0) { g_err = "dm_get_scene_name: empty buffer"; return fail(); }
    std::snprintf(out, static_cast<size_t>(cap), "%s", name);
    return 0;
}
int dm_get_static(dm_handle* h, int kind, double* out) {
    const std::vector<double>* v = nullptr;
    switch (kind) {
        case DM_STATE_OFFSET: v = &h->st_off; break; case DM_STATE_SCALE: v = &h->st_scale; break; case DM_ACTION_OFFSET: v = &h->act_off; break;
        case DM_ACTION_SCALE: v = &h->act_scale; break; case DM_ACTION_BOUND_MIN: v = &h->act_min; break; case DM_ACTION_BOUND_MAX: v = &h->act_max; break;
        case DM_STATE_NORM_GROUPS: v = &h->st_groups; break; default: g_err = "dm_get_static: bad kind"; return fail();
    }
    std::copy(v->begin(), v->end(), out);
    return 0;
}
void* dm_stream(dm_handle* h) { return h->stream; }
int dm_sync(dm_handle* h) { DM_DEVICE(h); DM_CUDA(cudaStreamSynchronize(h->stream)); return 0; }
int dm_set_mode(dm_handle* h, int mode) {
    h->mode = mode;
    h->hm.test_mode = mode;
    // the task scenes read the mode inside the kernels (test-mode get-ups, rewards)
    return task_scene(h) ? upload_model(h, offsetof(dmk::DevModel, test_mode), sizeof(int)) : 0;
}
// cRLSceneSimChar::SetSampleCount -> UpdateTimerParams (RLSceneSimChar.cpp:223-227,330-347): the episode time limits move from
// (time_lim_min, time_lim_max) to (time_end_lim_min, time_end_lim_max) with lerp = clamp(count / anneal_samples, 0, 1)^4.
int dm_set_sample_count(dm_handle* h, long long count) {
    const dmh::SceneConfig& c = h->sa.cfg;
    if (c.anneal_samples <= 0) return 0;
    double t = static_cast<double>(count) / static_cast<double>(c.anneal_samples);
    t = std::min(std::max(t, 0.0), 1.0);
    const double lerp = std::pow(t, 4.0);
    auto mix = [lerp](double a, double b) { return (a == b) ? a : (1.0 - lerp) * a + lerp * b; };   // cMathUtil::Lerp; a == b keeps infinities finite-safe
    h->hm.time_lim_min = mix(c.time_lim_min, c.time_end_lim_min);
    h->hm.time_lim_max = mix(c.time_lim_max, c.time_end_lim_max);
    return upload_time_limits(h);   // the reset kernel reads the limits from the model blob, stream-ordered
}
// Episode time limits set directly (both train-mode bounds): bench.py and tests that want a fixed limit without the annealing schedule.
int dm_set_time_limits(dm_handle* h, double tmin, double tmax) {
    if (!(tmin > 0.0) || !(tmax >= tmin)) { g_err = "dm_set_time_limits: need 0 < min <= max"; return fail(); }
    h->hm.time_lim_min = tmin; h->hm.time_lim_max = tmax;
    return upload_time_limits(h);
}
int dm_get_time_limits(dm_handle* h, double* out) {
    out[0] = h->hm.time_lim_min; out[1] = h->hm.time_lim_max; out[2] = h->hm.time_end_lim_max;
    return 0;
}

int dm_reset_clips(dm_handle* h, int force_all, const int* h_clip, const double* kt, const double* mt, const double* th) {
    DM_DEVICE(h);
    if (h_clip) {
        if (!task_scene(h)) { g_err = "dm_reset_clips: clip ids can only be injected in the AMP task scenes"; return fail(); }
        for (int e = 0; e < h->num_envs; ++e)
            if (h_clip[e] < 0 || h_clip[e] >= h->ctab.num_clips) { g_err = "dm_reset_clips: clip id out of range"; return fail(); }
    }
    const double* src[3] = {kt, mt, th};
    for (int k = 0; k < 3; ++k) if (src[k] && stage_envs(h, src[k], h->d_inj[k])) return 1;
    if (h_clip && stage_envs(h, h_clip, h->d_clip_inj)) return 1;
    if (h->d_push) {   // the environments about to be reset lose their push (cWorld::Reset clears its perturbations)
        dmk::dm_push_clear_kernel<<<(h->num_envs + 127) / 128, 128, 0, h->stream>>>(h->st, h->d_push, force_all);
        if (launched(h)) return 1;
    }
    if (launch_reset(h, force_all, kt ? h->d_inj[0] : nullptr, mt ? h->d_inj[1] : nullptr, th ? h->d_inj[2] : nullptr, h_clip ? h->d_clip_inj : nullptr)) return 1;
    if (h->dyn_random) {   // the restarted environments' factors for their new episode (the others' draws do not change)
        dmk::dm_dyn_draw_kernel<<<(h->num_envs + 127) / 128, 128, 0, h->stream>>>(h->st, h->d_dyn, h->dyn_rand);
        if (launched(h)) return 1;
    }
    if (!task_scene(h)) return 0;
    // cSceneTargetAMP::Reset's own part for the environments that were just reset
    dmk::dm_task_reset_kernel<<<(h->padded_envs + 127) / 128, 128, 0, h->stream>>>(h->d_model, h->st, h->padded_envs);
    return launched(h);
}
int dm_reset(dm_handle* h, int force_all, const double* kt, const double* mt, const double* th) { return dm_reset_clips(h, force_all, nullptr, kt, mt, th); }
int dm_get_clip_table(dm_handle* h, int* num_clips, double* h_dur, double* h_cdf) {
    const int n = static_cast<int>(h->sa.clips.size());
    if (num_clips) *num_clips = n;
    for (int c = 0; c < n; ++c) { if (h_dur) h_dur[c] = h->sa.clips[c].duration(); if (h_cdf) h_cdf[c] = h->sa.clip_cdf[c]; }
    return 0;
}
int dm_set_action(dm_handle* h, const float* d_actions) {
    DM_DEVICE(h);
    const int total = h->num_envs * h->hm.nl;
    dmk::dm_set_action_kernel<<<(total + 127) / 128, 128, 0, h->stream>>>(h->d_model, h->st, d_actions, h->num_envs);
    return launched(h);
}
int dm_update(dm_handle* h, double dt, int n_updates) {
    DM_DEVICE(h);
    if (h->d_push_sched) {   // the schedule refills the empty entries first, on the device: no host synchronisation
        dmk::dm_push_schedule_kernel<<<(h->num_envs + 127) / 128, 128, 0, h->stream>>>(h->st, h->d_push, h->d_push_sched, h->push_sched);
        if (launched(h)) return 1;
    }
    return launch_step(h, dt, n_updates);
}
// the handle's push table, every entry empty (the padding environments never run: theirs stay empty)
static int alloc_push_table(dm_handle* h) {
    if (alloc_buffer(h, &h->d_push, static_cast<size_t>(h->padded_envs))) return 1;
    std::vector<dmk::DevPush> none(static_cast<size_t>(h->padded_envs));
    for (auto& p : none) { p.force[0] = p.force[1] = p.force[2] = 0.f; p.body = -1; p.start = 0.0; p.duration = 0.0; }
    DM_CUDA(cudaMemcpyAsync(h->d_push, none.data(), none.size() * sizeof(dmk::DevPush), cudaMemcpyHostToDevice, h->stream));
    DM_CUDA(cudaStreamSynchronize(h->stream));
    return 0;
}
int dm_set_pushes(dm_handle* h, const int32_t* h_body, const float* h_force, const double* h_start, const double* h_duration) {
    DM_DEVICE(h);
    if (!h_body || !h_force || !h_start || !h_duration) { g_err = "dm_set_pushes: every array is required"; return fail(); }
    if (h->d_push_sched) { g_err = "dm_set_pushes: the handle has a push schedule (dm_set_push_schedule), which owns its push table"; return fail(); }
    const int N = h->num_envs, nl = h->hm.nl;
    std::vector<dmk::DevPush> tab(static_cast<size_t>(N));
    for (int e = 0; e < N; ++e) {
        auto refuse = [&](const char* what) { g_err = std::string("dm_set_pushes: environment ") + std::to_string(e) + ": " + what; return fail(); };
        if (h_body[e] < -1 || h_body[e] >= nl) return refuse(("body out of [-1, " + std::to_string(nl) + ")").c_str());
        for (int k = 0; k < 3; ++k) if (!std::isfinite(h_force[3 * e + k])) return refuse("force is not finite");
        if (!std::isfinite(h_start[e])) return refuse("start is not finite");
        if (!std::isfinite(h_duration[e]) || h_duration[e] < 0.0) return refuse("duration is negative or not finite");
        dmk::DevPush& p = tab[e];
        p.force[0] = h_force[3 * e]; p.force[1] = h_force[3 * e + 1]; p.force[2] = h_force[3 * e + 2];
        p.body = h_body[e]; p.start = h_start[e]; p.duration = h_duration[e];
    }
    if (h->d_push == nullptr && alloc_push_table(h)) return 1;
    DM_CUDA(cudaMemcpyAsync(h->d_push, tab.data(), tab.size() * sizeof(dmk::DevPush), cudaMemcpyHostToDevice, h->stream));
    DM_CUDA(cudaStreamSynchronize(h->stream));   // the staging vector is pageable
    return 0;
}
int dm_set_push_schedule(dm_handle* h, const int32_t* h_bodies, int n_bodies, const double* force2, const double* duration2, const double* gap2) {
    DM_DEVICE(h);
    auto refuse = [](const std::string& what) { g_err = "dm_set_push_schedule: " + what; return fail(); };
    if (h->d_push && !h->d_push_sched) return refuse("the handle has pushes set by dm_set_pushes, which own its push table");
    if (!h_bodies || !force2 || !duration2 || !gap2) return refuse("every array is required");
    if (n_bodies < 1 || n_bodies > dmk::kMaxPushBodies) return refuse("n_bodies " + std::to_string(n_bodies) + " outside [1, 32]");
    dmk::PushSchedule P;
    std::memset(&P, 0, sizeof(P));   // padding included: the state header hashes the bytes
    P.n_bodies = n_bodies;
    for (int i = 0; i < n_bodies; ++i) {
        if (h_bodies[i] < 0 || h_bodies[i] >= h->hm.nl)
            return refuse("h_bodies[" + std::to_string(i) + "] = " + std::to_string(h_bodies[i]) + " outside [0, " + std::to_string(h->hm.nl) + ")");
        P.bodies[i] = h_bodies[i];
    }
    const std::pair<const char*, const double*> bounds[3] = {{"force2", force2}, {"duration2", duration2}, {"gap2", gap2}};
    for (const auto& b : bounds) {
        const double lo = b.second[0], hi = b.second[1];
        if (!std::isfinite(lo) || !std::isfinite(hi)) return refuse(std::string(b.first) + ": a bound is not finite");
        if (lo < 0.0 || hi < 0.0) return refuse(std::string(b.first) + ": a bound is negative");
        if (lo > hi) return refuse(std::string(b.first) + ": lo > hi");
    }
    for (int k = 0; k < 2; ++k) { P.force[k] = force2[k]; P.duration[k] = duration2[k]; P.gap[k] = gap2[k]; }
    P.seed = h->seed ^ dmk::kPushSeedKey; P.env_base = h->env_offset;
    if (h->d_push_sched == nullptr) {   // zeroed: reset counter 0 never matches a live environment's (dm_create's reset makes it 1)
        if (alloc_push_table(h) || alloc_buffer(h, &h->d_push_sched, static_cast<size_t>(h->padded_envs) * dmk::kPushSchedDoubles, kZeroed)) return 1;
    }
    h->push_sched = P;
    return 0;
}
int dm_get_push_table(dm_handle* h, int32_t* h_body, float* h_force, double* h_window, double* h_sched) {
    DM_DEVICE(h);
    if (h_sched && !h->d_push_sched) { g_err = "dm_get_push_table: the handle has no push schedule"; return fail(); }
    const size_t N = static_cast<size_t>(h->num_envs);
    std::vector<dmk::DevPush> tab(N);
    for (auto& p : tab) { p.force[0] = p.force[1] = p.force[2] = 0.f; p.body = -1; p.start = 0.0; p.duration = 0.0; }
    if (h->d_push) DM_CUDA(cudaMemcpyAsync(tab.data(), h->d_push, N * sizeof(dmk::DevPush), cudaMemcpyDeviceToHost, h->stream));
    if (h_sched) DM_CUDA(cudaMemcpyAsync(h_sched, h->d_push_sched, N * dmk::kPushSchedDoubles * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    DM_CUDA(cudaStreamSynchronize(h->stream));
    for (size_t e = 0; e < N; ++e) {
        if (h_body) h_body[e] = tab[e].body;
        if (h_force) for (int k = 0; k < 3; ++k) h_force[3 * e + k] = tab[e].force[k];
        if (h_window) { h_window[2 * e] = tab[e].start; h_window[2 * e + 1] = tab[e].duration; }
    }
    return 0;
}
int dm_get_pushes(dm_handle* h, int32_t* h_body) {
    DM_DEVICE(h);
    if (h->d_push == nullptr) { std::fill(h_body, h_body + h->num_envs, -1); return 0; }
    std::vector<dmk::DevPush> tab(static_cast<size_t>(h->num_envs));
    DM_CUDA(cudaMemcpyAsync(tab.data(), h->d_push, tab.size() * sizeof(dmk::DevPush), cudaMemcpyDeviceToHost, h->stream));
    DM_CUDA(cudaStreamSynchronize(h->stream));
    for (int e = 0; e < h->num_envs; ++e) h_body[e] = tab[e].body;
    return 0;
}
// ---- dynamics (dm_dynamics.cuh)
namespace {
// a fixed leaf lumped into its parent's composite body by the step kernel (dm_step.cu: the dynamics tree)
int lumped_parent(const dmk::DevModel& M, int l) {
    const dmk::DevLink& L = M.link[l];
    return (L.ndof == 0 && L.nchild == 0 && L.parent >= 0 && M.link[L.parent].ndof > 0) ? L.parent : -1;
}
float link_mass_counted(const dmk::DevModel& M, int l) { return M.link[l].shape != 0 ? M.link[l].mass : 0.f; }   // CharModel::total_mass skips shapeless bodies
// the table and the empty push table of the dynamics kernel, every entry the plain model
int alloc_dyn_table(dm_handle* h) {
    const dmk::DevModel& M = h->hm;
    if (alloc_buffer(h, &h->d_dyn, static_cast<size_t>(h->padded_envs))) return 1;
    if (h->d_push_none == nullptr) {
        if (alloc_buffer(h, &h->d_push_none, static_cast<size_t>(h->padded_envs))) return 1;
        std::vector<dmk::DevPush> none(static_cast<size_t>(h->padded_envs));
        for (auto& p : none) { p.force[0] = p.force[1] = p.force[2] = 0.f; p.body = -1; p.start = 0.0; p.duration = 0.0; }
        DM_CUDA(cudaMemcpyAsync(h->d_push_none, none.data(), none.size() * sizeof(dmk::DevPush), cudaMemcpyHostToDevice, h->stream));
        DM_CUDA(cudaStreamSynchronize(h->stream));
    }
    std::vector<dmk::DevDyn> unit(static_cast<size_t>(h->padded_envs));
    std::vector<float> mass(M.nl);
    for (int l = 0; l < M.nl; ++l) mass[l] = link_mass_counted(M, l);
    for (auto& d : unit) {
        for (int k = 0; k < dmk::kDynFloats; ++k) d.f[k] = (k < dmk::kDTotalMass) ? 1.f : 0.f;
        d.f[dmk::kDTotalMass] = dmk::dyn_total_mass(mass.data(), M.nl, d.f);
    }
    DM_CUDA(cudaMemcpyAsync(h->d_dyn, unit.data(), unit.size() * sizeof(dmk::DevDyn), cudaMemcpyHostToDevice, h->stream));
    DM_CUDA(cudaStreamSynchronize(h->stream));
    return 0;
}
const char* const kDynKindNames[dmk::kDynKinds] = {"friction", "kp", "kd", "torque_limit", "mass"};
}  // namespace
int dm_set_dynamics(dm_handle* h, const float* h_factors) {
    DM_DEVICE(h);
    auto refuse = [](const std::string& what) { g_err = "dm_set_dynamics: " + what; return fail(); };
    if (!h_factors) return refuse("h_factors is required");
    if (h->dyn_random) return refuse("the handle's dynamics are randomised (dm_set_dynamics_randomization), which owns its table");
    const dmk::DevModel& M = h->hm;
    const int N = h->num_envs, nl = M.nl, row = 4 + nl;
    std::vector<float> mass(nl);
    for (int l = 0; l < nl; ++l) mass[l] = link_mass_counted(M, l);
    std::vector<dmk::DevDyn> tab(static_cast<size_t>(h->padded_envs));
    for (int e = 0; e < N; ++e) {
        const float* f = h_factors + static_cast<size_t>(e) * row;
        const std::string env = "environment " + std::to_string(e) + ": ";
        for (int j = 0; j < 4; ++j)
            if (!std::isfinite(f[j]) || f[j] < 0.f) return refuse(env + kDynKindNames[j] + " " + std::to_string(f[j]) + " is not finite and >= 0");
        for (int l = 0; l < nl; ++l)
            if (!std::isfinite(f[4 + l]) || !(f[4 + l] > 0.f))
                return refuse(env + "mass of link " + std::to_string(l) + " " + std::to_string(f[4 + l]) + " is not finite and > 0");
        for (int l = 0; l < nl; ++l) {
            const int p = lumped_parent(M, l);
            if (p >= 0 && f[4 + l] != f[4 + p])
                return refuse(env + "mass of link " + std::to_string(l) + " differs from its parent link " + std::to_string(p) +
                              "'s: a fixed leaf is part of its parent's composite body");
        }
        dmk::DevDyn& d = tab[e];
        for (int k = 0; k < dmk::kDynFloats; ++k) d.f[k] = (k < dmk::kDTotalMass) ? 1.f : 0.f;
        for (int j = 0; j < row; ++j) d.f[j] = f[j];
        d.f[dmk::kDTotalMass] = dmk::dyn_total_mass(mass.data(), nl, d.f);
    }
    for (int e = N; e < h->padded_envs; ++e) tab[e] = tab[N - 1];   // padding: never simulated
    if (h->d_dyn == nullptr && alloc_dyn_table(h)) return 1;
    DM_CUDA(cudaMemcpyAsync(h->d_dyn, tab.data(), tab.size() * sizeof(dmk::DevDyn), cudaMemcpyHostToDevice, h->stream));
    DM_CUDA(cudaStreamSynchronize(h->stream));   // the staging vector is pageable
    return 0;
}
int dm_get_dynamics(dm_handle* h, float* d_out) {
    DM_DEVICE(h);
    if (!d_out) { g_err = "dm_get_dynamics: d_out is required"; return fail(); }
    if (h->d_dyn == nullptr) { g_err = "dm_get_dynamics: the handle has no dynamics table (dm_set_dynamics, dm_set_dynamics_randomization)"; return fail(); }
    const size_t row = static_cast<size_t>(4 + h->hm.nl) * sizeof(float);
    DM_CUDA(cudaMemcpy2DAsync(d_out, row, h->d_dyn, sizeof(dmk::DevDyn), row, static_cast<size_t>(h->num_envs), cudaMemcpyDeviceToDevice, h->stream));
    return 0;
}
int dm_set_dynamics_randomization(dm_handle* h, const double* lohi) {
    DM_DEVICE(h);
    auto refuse = [](const std::string& what) { g_err = "dm_set_dynamics_randomization: " + what; return fail(); };
    if (!lohi) return refuse("lohi is required");
    if (h->d_dyn && !h->dyn_random) return refuse("the handle has factors set by dm_set_dynamics, which own its table");
    for (int k = 0; k < dmk::kDynKinds; ++k) {
        const double lo = lohi[2 * k], hi = lohi[2 * k + 1];
        const std::string kind = kDynKindNames[k];
        if (!std::isfinite(lo) || !std::isfinite(hi)) return refuse(kind + ": a bound is not finite");
        if (lo < 0.0 || hi < 0.0) return refuse(kind + ": a bound is negative");
        if (lo > hi) return refuse(kind + ": lo > hi");
        if (k == 4 && !(lo > 0.0)) return refuse(kind + ": lo must be > 0");
    }
    const dmk::DevModel& M = h->hm;
    dmk::DynRand R;
    std::memset(&R, 0, sizeof(R));   // padding included: the state header hashes the bytes
    for (int k = 0; k < 2 * dmk::kDynKinds; ++k) R.lohi[k] = lohi[k];
    R.seed = h->seed ^ dmk::kDynSeedKey; R.env_base = h->env_offset; R.nl = M.nl;
    for (int l = 0; l < 32; ++l) { R.leaf_parent[l] = l < M.nl ? lumped_parent(M, l) : -1; R.link_mass[l] = l < M.nl ? link_mass_counted(M, l) : 0.f; }
    if (h->d_dyn == nullptr && alloc_dyn_table(h)) return 1;
    h->dyn_rand = R; h->dyn_random = true;
    dmk::dm_dyn_draw_kernel<<<(h->num_envs + 127) / 128, 128, 0, h->stream>>>(h->st, h->d_dyn, h->dyn_rand);
    return launched(h);
}
int dm_set_env_order(dm_handle* h, int on) {
    DM_DEVICE(h);
    // placement by contact load pays where two environments share a warp (W = 16).  With one environment per warp (dog3d, W = 32) it measured
    // slower (dog trot, 2048 environments, H100 at 700 W: 0.741 M against 0.753 M policy steps/s), and so did the W = 32 kernels that carried
    // the key and the indirection: they keep index placement.
    h->st.order = (on && h->W == 16) ? h->d_order : nullptr;
    return 0;
}
int dm_plan_env_order(const int* keys, int n_padded, int tiles, int W, int* order) {
    if (!keys || !order || (W != 16 && W != 32) || tiles <= 0 || tiles % (32 / W) != 0 || n_padded <= 0 || n_padded % tiles != 0) {
        g_err = "dm_plan_env_order: bad arguments";
        return fail();
    }
    std::vector<int> sorted(n_padded);
    std::iota(sorted.begin(), sorted.end(), 0);
    std::stable_sort(sorted.begin(), sorted.end(), [&](int a, int b) { return dmk::env_load_bucket(keys[a]) < dmk::env_load_bucket(keys[b]); });
    for (int r = 0; r < n_padded; ++r) order[dmk::env_order_slot(r, n_padded, tiles, W)] = sorted[r];
    return 0;
}
int dm_get_env_order(dm_handle* h, int* h_plan3, int* h_keys, int* h_order) {
    DM_DEVICE(h);
    if (h_plan3) { h_plan3[0] = h->padded_envs; h_plan3[1] = h->tiles; h_plan3[2] = h->W; }
    DM_CUDA(cudaStreamSynchronize(h->stream));
    if (h_keys) DM_CUDA(cudaMemcpy(h_keys, h->st.load, sizeof(int) * h->padded_envs, cudaMemcpyDeviceToHost));
    if (h_order && h->st.order) DM_CUDA(cudaMemcpy(h_order, h->st.order, sizeof(int) * h->padded_envs, cudaMemcpyDeviceToHost));
    else if (h_order) std::iota(h_order, h_order + h->padded_envs, 0);
    return 0;
}
static int launch_task_observe(dm_handle* h, float* d_goal, float* d_reward) {
    dmk::dm_task_observe_kernel<<<(h->num_envs + 127) / 128, 128, 0, h->stream>>>(h->d_model, h->st, d_goal, d_reward, h->num_envs);
    return launched(h);
}
int dm_observe(dm_handle* h, float* d_state, float* d_reward) {
    DM_DEVICE(h);
    const bool task = task_scene(h);   // the task scenes replace CalcReward (SceneTargetAMP.cpp:3-80, SceneHeadingAMP.cpp:3-48)
    float* d_imitate_reward = task ? nullptr : d_reward;
    if ((d_state != nullptr || d_imitate_reward != nullptr) && launch_observe(h, d_state, d_imitate_reward)) return 1;
    if (task && d_reward != nullptr) return launch_task_observe(h, nullptr, d_reward);
    return 0;
}
int dm_record_state(dm_handle* h, float* d_out) { return dm_observe(h, d_out, nullptr); }
int dm_record_pose(dm_handle* h, float* d_pose, float* d_vel) {
    DM_DEVICE(h);
    if (d_pose == nullptr && d_vel == nullptr) return 0;
    return launch_pose(h, d_pose, d_vel);
}
int dm_render_poses(dm_handle* h, int n_views, const float* d_pose, const dm_camera* cam, int width, int height, uint8_t* d_rgb, int16_t* d_ids) {
    DM_DEVICE(h);
    auto refuse = [](const std::string& what) { g_err = "dm_render_poses: " + what; return fail(); };
    if (n_views < 1 || n_views > 65535) return refuse("n_views " + std::to_string(n_views) + " outside [1, 65535]");
    if (width < 16 || width > 4096) return refuse("width " + std::to_string(width) + " outside [16, 4096]");
    if (height < 16 || height > 4096) return refuse("height " + std::to_string(height) + " outside [16, 4096]");
    if (d_pose == nullptr) return refuse("d_pose is NULL");
    if (d_rgb == nullptr && d_ids == nullptr) return refuse("d_rgb and d_ids are both NULL");
    if (cam == nullptr) return refuse("cam is NULL");
    const char* names[5] = {"yaw", "pitch", "distance", "target_height", "fov_y"};
    const float vals[5] = {cam->yaw, cam->pitch, cam->distance, cam->target_height, cam->fov_y};
    for (int k = 0; k < 5; ++k)
        if (!std::isfinite(vals[k])) return refuse(std::string("camera ") + names[k] + " is not finite");
    if (!(cam->distance > 0.f)) return refuse("camera distance " + std::to_string(cam->distance) + " <= 0");
    if (!(cam->fov_y > 0.f && cam->fov_y < static_cast<float>(M_PI))) return refuse("camera fov_y " + std::to_string(cam->fov_y) + " outside (0, pi)");
    // the camera basis in double: fwd from the eye to the target, right = fwd x up normalised (cos yaw, 0, -sin yaw), up = right x fwd
    const double cy = std::cos(cam->yaw), sy = std::sin(cam->yaw), cp = std::cos(cam->pitch), sp = std::sin(cam->pitch);
    const V3 back(cp * sy, sp, cp * cy), right(cy, 0.0, -sy);
    const V3 fwd = -1.0 * back, up(right.y * fwd.z - right.z * fwd.y, right.z * fwd.x - right.x * fwd.z, right.x * fwd.y - right.y * fwd.x);
    dmk::RenderCam rc;
    put3(rc.back, back, cam->distance); put3(rc.fwd, fwd); put3(rc.right, right); put3(rc.up, up);
    rc.tan_y = static_cast<float>(std::tan(0.5 * cam->fov_y));
    rc.tan_x = static_cast<float>(std::tan(0.5 * cam->fov_y) * width / height);
    rc.target_height = cam->target_height;
    const int T = dmk::kRenderTile;
    const dim3 grid(((width + T - 1) / T) * ((height + T - 1) / T), n_views);
    dmk::dm_render_kernel<<<grid, T * T, 0, h->stream>>>(h->d_model, d_pose, width, height, rc, d_rgb, d_ids);
    DM_CUDA(cudaGetLastError());
    return 0;
}
int dm_record_kin_pose(dm_handle* h, float* d_pose) {
    DM_DEVICE(h);
    if (d_pose == nullptr) return 0;
    const int threads = 256, total = h->num_envs * h->hm.nl;
    dmk::kKinPoseKernels[task_scene(h)]<<<(total + threads - 1) / threads, threads, 0, h->stream>>>(h->d_model, h->st, h->d_frame_times, h->d_frames,
                                                                                                   h->d_frame_vel, d_pose, h->num_envs);
    return launched(h);
}
int dm_pose_error(dm_handle* h, int T, int n, const float* d_a, const float* d_r, const int32_t* d_len, float* d_lock, float* d_dtw) {
    DM_DEVICE(h);
    auto refuse = [](const std::string& what) { g_err = "dm_pose_error: " + what; return fail(); };
    if (T < 1) return refuse("T " + std::to_string(T) + " < 1");
    if (n < 1) return refuse("n " + std::to_string(n) + " < 1");
    if (d_a == nullptr) return refuse("d_a is NULL");
    if (d_r == nullptr) return refuse("d_r is NULL");
    if (d_len == nullptr) return refuse("d_len is NULL");
    const int nj = h->hm.nl - 1;
    if (nj < 1) return refuse("the character has no joint besides the root");
    if (d_lock == nullptr && d_dtw == nullptr) return 0;
    const size_t rows = static_cast<size_t>(T) * n, F = 3 * static_cast<size_t>(nj);
    if ((rows + dmk::kPoseFeatureThreads / 32 - 1) / (dmk::kPoseFeatureThreads / 32) > 0x7fffffffu) return refuse("T x n too large");
    // scratch from the stream's memory pool, released in stream order: both sequences' features [2][n][T][F] and the DP's boundary rows [n][T]
    float* scratch = nullptr;
    DM_CUDA(cudaMallocAsync(&scratch, sizeof(float) * (2 * rows * F + rows), h->stream));
    const unsigned fblocks = static_cast<unsigned>((rows + dmk::kPoseFeatureThreads / 32 - 1) / (dmk::kPoseFeatureThreads / 32));
    dmk::dm_pose_feature_kernel<<<dim3(fblocks, 2), dmk::kPoseFeatureThreads, 0, h->stream>>>(h->d_model, d_a, d_r, T, n, scratch);
    const size_t smem = dmk::dm_pose_dtw_smem(nj);
    const dmk::PoseDtwKernel kern = dmk::kPoseDtwKernels[nj <= 15 ? 0 : 1];
    cudaError_t err = cudaGetLastError();
    if (err == cudaSuccess) err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (err == cudaSuccess) {
        kern<<<n, dmk::kPoseDtwThreads, smem, h->stream>>>(scratch, T, n, nj, d_len, scratch + 2 * rows * F, d_lock, d_dtw);
        err = cudaGetLastError();
    }
    DM_CUDA(cudaFreeAsync(scratch, h->stream));
    DM_CUDA(err);
    return 0;
}
// cSceneImitate::CalcRewardImitate in every scene: in the AMP task scenes (where CalcReward is the task reward) against the environment's
// active clip of the dataset -- BASELINE.json config 5 records it beside the AMP observations.
int dm_calc_reward_imitate(dm_handle* h, float* d_out) {
    DM_DEVICE(h);
    return launch_observe(h, nullptr, d_out);
}
int dm_record_goal(dm_handle* h, float* d_out) {
    if (!task_scene(h)) return 0;
    DM_DEVICE(h);
    return launch_task_observe(h, d_out, nullptr);
}
int dm_goal_host(dm_handle* h, float* h_out) {
    if (!task_scene(h)) return 0;
    DM_DEVICE(h);
    if (launch_task_observe(h, h->d_goal, nullptr)) return 1;
    const size_t gbytes = static_cast<size_t>(h->num_envs) * goal_size(h->hm) * sizeof(float);
    DM_CUDA(cudaMemcpyAsync(h->p_goal, h->d_goal, gbytes, cudaMemcpyDeviceToHost, h->stream));
    DM_CUDA(cudaStreamSynchronize(h->stream));
    std::memcpy(h_out, h->p_goal, gbytes);
    return 0;
}
// test hooks of the task scenes: the environment's task block (dm_task.cuh: TaskSlot) and the scene constants as the device sees them
int dm_get_task_state(dm_handle* h, int env, double* h_out) {
    if (!task_scene(h)) { g_err = "dm_get_task_state: not a task scene"; return fail(); }
    DM_DEVICE(h);
    DM_CUDA(cudaStreamSynchronize(h->stream));
    DM_CUDA(cudaMemcpy(h_out, h->st.task + static_cast<size_t>(env) * dmk::kTaskDoubles, dmk::kTaskDoubles * sizeof(double), cudaMemcpyDeviceToHost));
    DM_CUDA(cudaMemcpy(h_out + dmk::kTaskDoubles, h->st.taskx + static_cast<size_t>(env) * dmk::kTaskExtDoubles, dmk::kTaskExtDoubles * sizeof(double), cudaMemcpyDeviceToHost));
    return 0;
}
int dm_set_task_state(dm_handle* h, int env, const double* h_in) {
    if (!task_scene(h)) { g_err = "dm_set_task_state: not a task scene"; return fail(); }
    DM_DEVICE(h);
    DM_CUDA(cudaStreamSynchronize(h->stream));
    DM_CUDA(cudaMemcpy(h->st.task + static_cast<size_t>(env) * dmk::kTaskDoubles, h_in, dmk::kTaskDoubles * sizeof(double), cudaMemcpyHostToDevice));
    DM_CUDA(cudaMemcpy(h->st.taskx + static_cast<size_t>(env) * dmk::kTaskExtDoubles, h_in + dmk::kTaskDoubles, dmk::kTaskExtDoubles * sizeof(double), cudaMemcpyHostToDevice));
    return 0;
}
int dm_get_task_params(dm_handle* h, double* o, unsigned long long* stream) {
    const dmk::TaskParams& T = h->hm.task;
    o[0] = h->hm.task_kind; o[1] = T.timer_min; o[2] = T.timer_max; o[3] = T.max_target_dist; o[4] = T.target_succ_dist; o[5] = T.tar_fail_dist; o[6] = T.pos_reward_scale;
    o[7] = T.max_heading_turn_rate; o[8] = T.sharp_turn_prob; o[9] = T.speed_change_prob; o[10] = T.tar_speed_min; o[11] = T.tar_speed_max; o[12] = T.vel_reward_scale;
    o[13] = T.tar_speed; o[14] = T.enable_min_tar_vel; o[15] = 0;
    {   // dm_task_ext.cuh constants, in the order tests/task_shim.cpp reads them
        const dmk::TaskExtParams& X = h->hm.taskx;
        double* q = o + 16;
        q[0] = X.getup_time; q[1] = X.getup_height_root; q[2] = X.getup_height_head; q[3] = X.recover_episode_prob;
        for (int k = 0; k < 3; ++k) { q[4 + k] = X.target_min[k]; q[7 + k] = X.target_max[k]; }
        q[10] = X.target_radius; q[11] = X.hit_reset_time; q[12] = X.tar_reward_scale; q[13] = X.hit_tar_speed; q[14] = X.init_hit_prob; q[15] = X.tar_far_prob; q[16] = X.tar_near_dist;
        q[17] = X.head_id; q[18] = X.n_strike; q[23] = X.n_fail;
        for (int k = 0; k < 4; ++k) { q[19 + k] = X.strike_bodies[k]; q[24 + k] = X.fail_bodies[k]; }
        q[28] = q[29] = q[30] = q[31] = 0;
    }
    if (stream) { stream[0] = h->hm.task_seed; stream[1] = h->hm.env_id_base; }
    return 0;
}
int dm_record_amp_obs_agent(dm_handle* h, float* d_out) { DM_DEVICE(h); return launch_amp(h, d_out, 0, nullptr, nullptr); }
int dm_amp_obs_host(dm_handle* h, int expert, const double* h_kin_time, float* h_out) {
    DM_DEVICE(h);
    if (expert ? dm_record_amp_obs_expert(h, h_kin_time, h->d_amp) : dm_record_amp_obs_agent(h, h->d_amp)) return 1;
    const size_t bytes = static_cast<size_t>(h->num_envs) * h->hm.amp_obs_size * sizeof(float);
    DM_CUDA(cudaMemcpyAsync(h->p_amp, h->d_amp, bytes, cudaMemcpyDeviceToHost, h->stream));
    DM_CUDA(cudaStreamSynchronize(h->stream));
    std::memcpy(h_out, h->p_amp, bytes);
    return 0;
}
int dm_record_amp_obs_expert_clips(dm_handle* h, const int* h_clip, const double* h_kin_time, float* d_out) {
    DM_DEVICE(h);
    const bool task = task_scene(h);
    if (h_clip && !task) { g_err = "dm_record_amp_obs_expert_clips: clip ids can only be given in the AMP task scenes"; return fail(); }
    std::vector<int> ct(h->num_envs, 0);
    if (task) {   // cSceneImitateAMP::SampleExpertMotion: cClipsController::SampleMotionID per call (SceneImitateAMP.cpp:260-277)
        for (int e = 0; e < h->num_envs; ++e) {
            ct[e] = h_clip ? h_clip[e] : dmk::select_clip(h->ctab, dmk::task_u01(h->seed ^ 0x657870636c6970ull, h->env_offset + e, h->amp_calls));
            if (ct[e] < 0 || ct[e] >= h->ctab.num_clips) { g_err = "dm_record_amp_obs_expert_clips: clip id out of range"; return fail(); }
        }
    }
    std::vector<double> times(h->num_envs);
    if (h_kin_time) std::copy(h_kin_time, h_kin_time + h->num_envs, times.begin());
    else {   // cSceneImitateAMP::RecordAMPObsExpert draws U(0, duration) per call; here a counter-based stream per (seed, env, call)
        for (int e = 0; e < h->num_envs; ++e)
            times[e] = (task ? h->ctab.info[ct[e]].dur : h->hm.motion_dur) * dmk::task_u01(h->seed, h->env_offset + e, 0x51ed26ull + h->amp_calls);
    }
    if (!h_kin_time || (task && !h_clip)) h->amp_calls++;
    if (stage_envs(h, times.data(), h->d_inj[0]) || (task && stage_envs(h, ct.data(), h->d_clip_inj))) return 1;
    return launch_amp(h, d_out, 1, h->d_inj[0], task ? h->d_clip_inj : nullptr);
}
int dm_record_amp_obs_expert(dm_handle* h, const double* h_kin_time, float* d_out) { return dm_record_amp_obs_expert_clips(h, nullptr, h_kin_time, d_out); }
int dm_sample_amp_obs_expert(dm_handle* h, int rows, float* d_out, int* d_clip_out, double* d_time_out) {
    DM_DEVICE(h);
    if (rows < 1 || d_out == nullptr) { g_err = "dm_sample_amp_obs_expert: need rows >= 1 and an output buffer"; return fail(); }
    const dmk::AmpExpertKernel kern = dmk::kAmpExpertKernels[tile_index(h)][task_scene(h)];   // task scenes: the clip drawn from the dataset
    const int tiles = dmk::kPolicyBlock / h->W;
    kern<<<(rows + tiles - 1) / tiles, dmk::kPolicyBlock, 0, h->stream>>>(h->d_model, h->st, h->d_frame_times, h->d_frames, h->d_frame_vel, d_out, rows, h->seed,
                                                                          h->expert_samples, d_clip_out, d_time_out);
    h->expert_samples++;
    return launched(h);
}
int dm_expert_sample_count(dm_handle* h, const unsigned long long* h_set, unsigned long long* h_get) {
    if (h_get) *h_get = h->expert_samples;
    if (h_set) h->expert_samples = *h_set;
    return 0;
}
int dm_calc_reward(dm_handle* h, float* d_out) { return dm_observe(h, nullptr, d_out); }
int dm_get_flags(dm_handle* h, int32_t* d_flags) {
    DM_DEVICE(h);
    dmk::dm_flags_kernel<<<(h->num_envs + 127) / 128, 128, 0, h->stream>>>(h->st, d_flags, h->num_envs);
    return launched(h);
}
// true when the host pointer is page-locked (cudaMallocHost / cudaHostRegister): the copy engines can address it directly
static bool is_pinned_host(dm_handle* h, const void* p) {
    for (const auto& e : h->pin_cache) if (e.first == p) return e.second;
    cudaPointerAttributes at;
    bool pinned = false;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) cudaGetLastError();
    else pinned = at.type == cudaMemoryTypeHost;
    // a stale entry (buffer freed and the address reused with the other kind) costs performance only: cudaMemcpyAsync accepts pageable memory
    if (h->pin_cache.size() >= 32) h->pin_cache.clear();
    h->pin_cache.emplace_back(p, pinned);
    return pinned;
}
static inline double now_ms() {
    timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts);
    return 1e3 * static_cast<double>(ts.tv_sec) + 1e-6 * static_cast<double>(ts.tv_nsec);
}
int dm_set_timing(dm_handle* h, int on) {
    DM_DEVICE(h);
    if (on && !h->tev[0]) for (auto& e : h->tev) DM_CUDA(cudaEventCreate(&e));
    h->timing = on != 0;
    return 0;
}
int dm_step_host_timing(dm_handle* h, double* o) {
    DM_DEVICE(h);
    if (!h->timing || !h->tev[0]) { g_err = "dm_step_host_timing: call dm_set_timing(h, 1) before the dm_step_host to be measured"; return fail(); }
    float ms[4] = {0, 0, 0, 0};
    for (int k = 0; k < 4; ++k) DM_CUDA(cudaEventElapsedTime(&ms[k], h->tev[k], h->tev[k + 1]));
    for (int k = 0; k < 4; ++k) o[k] = ms[k];
    o[4] = h->host_ms[0]; o[5] = h->host_ms[1]; o[6] = h->host_ms[2]; o[7] = 0.0;
    return 0;
}
int dm_step_host(dm_handle* h, const float* h_actions, double dt, int n_updates, float* h_state, float* h_reward, int32_t* h_flags) {
    return dm_step_host_reset(h, h_actions, dt, n_updates, h_state, h_reward, h_flags, 0);
}
int dm_step_host_reset(dm_handle* h, const float* h_actions, double dt, int n_updates, float* h_state, float* h_reward, int32_t* h_flags, int reset_done) {
    DM_DEVICE(h);
    const size_t N = h->num_envs, A = h->hm.action_size, S = h->hm.state_size;
    // page-locked caller buffers are used as they are; pageable ones go through the handle's pinned staging buffers (one extra host copy)
    const bool pa = h_actions && is_pinned_host(h, h_actions), ps = h_state && is_pinned_host(h, h_state), pr = h_reward && is_pinned_host(h, h_reward),
               pf = h_flags && is_pinned_host(h, h_flags);
    const bool tm = h->timing;
    const double t0 = tm ? now_ms() : 0.0;
    double t_copy = 0.0;
    if (tm) DM_CUDA(cudaEventRecord(h->tev[0], h->stream));
    if (h_actions) {
        if (!pa) { const double c0 = tm ? now_ms() : 0.0; std::memcpy(h->p_act, h_actions, N * A * sizeof(float)); if (tm) t_copy += now_ms() - c0; }
        DM_CUDA(cudaMemcpyAsync(h->d_act, pa ? h_actions : h->p_act, N * A * sizeof(float), cudaMemcpyHostToDevice, h->stream));
        if (dm_set_action(h, h->d_act)) return 1;
    }
    if (tm) DM_CUDA(cudaEventRecord(h->tev[1], h->stream));
    if (n_updates > 0 && dm_update(h, dt, n_updates)) return 1;
    if (tm) DM_CUDA(cudaEventRecord(h->tev[2], h->stream));
    if (dm_observe(h, h_state ? h->d_obs : nullptr, h_reward ? h->d_rew : nullptr)) return 1;
    if (h_flags && dm_get_flags(h, h->d_flags4)) return 1;
    if (tm) DM_CUDA(cudaEventRecord(h->tev[3], h->stream));
    if (h_state) DM_CUDA(cudaMemcpyAsync(ps ? h_state : h->p_obs, h->d_obs, N * S * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    if (h_reward) DM_CUDA(cudaMemcpyAsync(pr ? h_reward : h->p_rew, h->d_rew, N * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    if (h_flags) DM_CUDA(cudaMemcpyAsync(pf ? h_flags : h->p_flags, h->d_flags4, N * 4 * sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
    if (tm) DM_CUDA(cudaEventRecord(h->tev[4], h->stream));
    const double t1 = tm ? now_ms() : 0.0;
    DM_CUDA(cudaStreamSynchronize(h->stream));
    const double t2 = tm ? now_ms() : 0.0;
    if (h_state && !ps) std::memcpy(h_state, h->p_obs, N * S * sizeof(float));
    if (h_reward && !pr) std::memcpy(h_reward, h->p_rew, N * sizeof(float));
    if (h_flags && !pf) std::memcpy(h_flags, h->p_flags, N * 4 * sizeof(int32_t));
    if (tm) { h->host_ms[0] = t1 - t0 - t_copy; h->host_ms[1] = t2 - t1; h->host_ms[2] = t_copy + (now_ms() - t2); }
    // the caller has the finished episodes' last state / reward / flags: restart them now, after the wait, so that the reset kernel runs
    // under the caller's own work and the next call finds the stream idle (the reference's caller resets right after IsEpisodeEnd)
    if (reset_done) return dm_reset(h, 0, nullptr, nullptr, nullptr);
    return 0;
}

// ---------------------------------------------------------------- multi-GPU exchange over NVLink peer memory (include/deepmimic_b200.h)
static size_t xchg_parity_floats(const dm_handle* h) { return static_cast<size_t>(h->x_world) * h->num_envs * (h->hm.state_size + 2); }
static float* xchg_plane(const dm_handle* h, const char* base, int parity, int plane /*0 obs 1 rew 2 done*/) {
    const size_t WN = static_cast<size_t>(h->x_world) * h->num_envs, S = h->hm.state_size;
    float* p = reinterpret_cast<float*>(const_cast<char*>(base) + h->x_data_off + static_cast<size_t>(parity) * h->x_parity_bytes);
    return plane == 0 ? p : (plane == 1 ? p + WN * S : p + WN * S + WN);
}
int dm_exchange_create(dm_handle* h, int rank, int world, void* h_ipc_out64) {
    DM_DEVICE(h);
    if (h->x_base) { g_err = "dm_exchange_create: the handle already has an exchange"; return fail(); }
    if (world < 1 || world > 8 || rank < 0 || rank >= world) { g_err = "dm_exchange_create: world must be 1..8 (one node) and 0 <= rank < world"; return fail(); }
    h->x_rank = rank; h->x_world = world;
    h->x_data_off = 1024;
    h->x_parity_bytes = ((xchg_parity_floats(h) * sizeof(float) + 255) / 256) * 256;
    const size_t bytes = h->x_data_off + 2 * h->x_parity_bytes;
    DM_CUDA(cudaMalloc(&h->x_base, bytes));
    DM_CUDA(cudaMemset(h->x_base, 0, bytes));
    DM_CUDA(cudaDeviceSynchronize());
    h->x_peer[rank] = h->x_base;
    cudaIpcMemHandle_t ipc;
    DM_CUDA(cudaIpcGetMemHandle(&ipc, h->x_base));
    static_assert(sizeof(ipc) == 64, "cudaIpcMemHandle_t is 64 bytes");
    std::memcpy(h_ipc_out64, &ipc, 64);
    return 0;
}
int dm_exchange_connect(dm_handle* h, const void* h_ipc_all) {
    DM_DEVICE(h);
    if (!h->x_base) { g_err = "dm_exchange_connect: call dm_exchange_create first"; return fail(); }
    for (int r = 0; r < h->x_world; ++r) {
        if (r == h->x_rank) continue;
        cudaIpcMemHandle_t ipc;
        std::memcpy(&ipc, static_cast<const char*>(h_ipc_all) + 64 * r, 64);
        void* p = nullptr;
        DM_CUDA(cudaIpcOpenMemHandle(&p, ipc, cudaIpcMemLazyEnablePeerAccess));
        h->x_peer[r] = static_cast<char*>(p);
    }
    return 0;
}
static dmk::XchgPeers xchg_peers(const dm_handle* h) {
    dmk::XchgPeers P{};
    P.n = h->x_world;
    for (int r = 0; r < h->x_world; ++r) P.f[r] = reinterpret_cast<dmk::XchgFlags*>(h->x_peer[r]);
    return P;
}
static const unsigned long long kXchgTimeoutNs = 20ull * 1000ull * 1000ull * 1000ull;
int dm_exchange_publish(dm_handle* h, long long step) {
    DM_DEVICE(h);
    if (!h->x_base) { g_err = "dm_exchange_publish: no exchange (dm_exchange_create / dm_exchange_connect)"; return fail(); }
    for (int r = 0; r < h->x_world; ++r) if (!h->x_peer[r]) { g_err = "dm_exchange_publish: peers are not connected"; return fail(); }
    const int par = static_cast<int>(step & 1);
    if (step >= 2 && h->x_world > 1) {   // the slot still holds step - 2: every rank must have released it
        dmk::dm_xchg_wait_kernel<<<1, 32, 0, h->stream>>>(reinterpret_cast<dmk::XchgFlags*>(h->x_base), h->x_world, 1, static_cast<unsigned long long>(step - 1), kXchgTimeoutNs);
        if (launched(h)) return 1;
    }
    dmk::ObsFan fan{};
    fan.n = h->x_world;
    const size_t N = h->num_envs, S = h->hm.state_size;
    int d = 0;
    for (int k = 0; k < h->x_world; ++k) {   // destination 0 = local, then the peers starting after this rank (spreads the first stores over the links)
        const int r = (h->x_rank + k) % h->x_world;
        fan.obs[d] = xchg_plane(h, h->x_peer[r], par, 0) + h->x_rank * N * S;
        fan.rew[d] = xchg_plane(h, h->x_peer[r], par, 1) + h->x_rank * N;
        fan.done[d] = xchg_plane(h, h->x_peer[r], par, 2) + h->x_rank * N;
        ++d;
    }
    if (task_scene(h)) { g_err = "dm_exchange_publish: the AMP task scenes are not wired to the exchange"; return fail(); }
    if (launch_observe_fan(h, fan)) return 1;
    dmk::dm_xchg_signal_kernel<<<1, 32, 0, h->stream>>>(xchg_peers(h), h->x_rank, 0, static_cast<unsigned long long>(step + 1));
    return launched(h);
}
int dm_exchange_acquire(dm_handle* h, long long step, float** d_obs, float** d_rew, float** d_done) {
    DM_DEVICE(h);
    if (!h->x_base) { g_err = "dm_exchange_acquire: no exchange"; return fail(); }
    if (h->x_world > 1) {
        dmk::dm_xchg_wait_kernel<<<1, 32, 0, h->stream>>>(reinterpret_cast<dmk::XchgFlags*>(h->x_base), h->x_world, 0, static_cast<unsigned long long>(step + 1), kXchgTimeoutNs);
        if (launched(h)) return 1;
    }
    const int par = static_cast<int>(step & 1);
    if (d_obs) *d_obs = xchg_plane(h, h->x_base, par, 0);
    if (d_rew) *d_rew = xchg_plane(h, h->x_base, par, 1);
    if (d_done) *d_done = xchg_plane(h, h->x_base, par, 2);
    return 0;
}
int dm_exchange_release(dm_handle* h, long long step) {
    DM_DEVICE(h);
    if (!h->x_base) { g_err = "dm_exchange_release: no exchange"; return fail(); }
    if (h->x_world == 1) return 0;
    dmk::dm_xchg_signal_kernel<<<1, 32, 0, h->stream>>>(xchg_peers(h), h->x_rank, 1, static_cast<unsigned long long>(step + 1));
    return launched(h);
}
int dm_exchange_status(dm_handle* h, int* status) {
    DM_DEVICE(h);
    if (!h->x_base) { g_err = "dm_exchange_status: no exchange"; return fail(); }
    DM_CUDA(cudaStreamSynchronize(h->stream));
    unsigned int s = 0;
    DM_CUDA(cudaMemcpy(&s, h->x_base + offsetof(dmk::XchgFlags, status), sizeof(s), cudaMemcpyDeviceToHost));
    *status = static_cast<int>(s);
    return 0;
}
int dm_exchange_destroy(dm_handle* h) {
    if (!h->x_base) return 0;
    cudaSetDevice(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    for (int r = 0; r < h->x_world; ++r) if (r != h->x_rank && h->x_peer[r]) { cudaIpcCloseMemHandle(h->x_peer[r]); }
    for (auto& p : h->x_peer) p = nullptr;
    cudaFree(h->x_base); h->x_base = nullptr; h->x_world = 0;
    return 0;
}

int dm_get_snapshot(dm_handle* h, int env, double* s) {
    DM_DEVICE(h);
    const auto& M = h->hm; const int nl = M.nl, ss = dmk::sim_stride(nl);
    std::vector<float> sim(ss), man(nl * dmk::kManifoldFloats); double tm[dmk::kTimeDoubles]; int fl[dmk::kFlagInts];
    DM_CUDA(cudaStreamSynchronize(h->stream));
    DM_CUDA(cudaMemcpy(sim.data(), h->st.sim + static_cast<size_t>(env) * ss, ss * sizeof(float), cudaMemcpyDeviceToHost));
    DM_CUDA(cudaMemcpy(man.data(), h->st.manifold + static_cast<size_t>(env) * nl * dmk::kManifoldFloats, man.size() * sizeof(float), cudaMemcpyDeviceToHost));
    DM_CUDA(cudaMemcpy(tm, h->st.time + static_cast<size_t>(env) * dmk::kTimeDoubles, sizeof(tm), cudaMemcpyDeviceToHost));
    DM_CUDA(cudaMemcpy(fl, h->st.flags + static_cast<size_t>(env) * dmk::kFlagInts, sizeof(fl), cudaMemcpyDeviceToHost));
    const SimOffsets so(nl);
    const SnapshotOffsets sn(nl);
    std::fill(s, s + sn.size, 0.0);
    for (int k = 0; k < 3; ++k) { s[k] = sim[k]; s[7 + k] = sim[8 + k]; s[10 + k] = sim[12 + k]; }
    for (int k = 0; k < 4; ++k) s[3 + k] = sim[4 + k];
    for (int j = 0; j < nl; ++j) {
        if (M.link[j].ndof > 0) for (int k = 0; k < 4; ++k) s[sn.jpos + 4 * j + k] = sim[so.jpos + 4 * j + k];
        else s[sn.jpos + 4 * j + 3] = 1.0;
        for (int k = 0; k < M.link[j].ndof; ++k) s[sn.jvel + 3 * j + k] = sim[so.jvel + 4 * j + k];
        for (int c = 0; c < 4; ++c) for (int k = 0; k < 12; ++k) s[sn.manifold + (j * 4 + c) * 12 + k] = man[j * dmk::kManifoldFloats + c * 12 + k];
        // PD target back to the joint-frame (w,x,y,z) convention
        const float* t = &sim[so.pd + 4 * j]; double* o = s + sn.pd + 4 * j;
        if (M.link[j].jtype == dmk::kJSpherical) {
            Quat cr(M.link[j].child_rot[3], M.link[j].child_rot[0], M.link[j].child_rot[1], M.link[j].child_rot[2]);
            Quat q = dmh::conj(cr) * Quat(t[3], t[0], t[1], t[2]) * cr;
            o[0] = q.w; o[1] = q.x; o[2] = q.y; o[3] = q.z;
        } else if (M.link[j].jtype == dmk::kJRevolute) o[0] = t[0];
    }
    double* q = s + sn.clocks;
    q[0] = tm[dmk::kTKin]; q[1] = tm[dmk::kTOrigin]; q[2] = tm[dmk::kTOrigin + 1]; q[3] = tm[dmk::kTOrigin + 2];
    for (int k = 0; k < 4; ++k) q[4 + k] = tm[dmk::kTOriginRot + k];
    q[8] = tm[dmk::kTCtrl]; q[9] = tm[dmk::kTInitOff]; q[10] = tm[dmk::kTPrevAct]; q[11] = fl[dmk::kFNeedAction]; q[12] = tm[dmk::kTTimer]; q[13] = tm[dmk::kTTimerMax];
    return 0;
}
int dm_set_snapshot(dm_handle* h, int env, const double* s) {
    DM_DEVICE(h);
    const auto& M = h->hm; const int nl = M.nl, ss = dmk::sim_stride(nl);
    std::vector<float> sim(ss, 0.f), man(nl * dmk::kManifoldFloats, 0.f); double tm[dmk::kTimeDoubles] = {0}; int fl[dmk::kFlagInts] = {0};
    DM_CUDA(cudaStreamSynchronize(h->stream));
    DM_CUDA(cudaMemcpy(fl, h->st.flags + static_cast<size_t>(env) * dmk::kFlagInts, sizeof(fl), cudaMemcpyDeviceToHost));
    for (int k = 0; k < 3; ++k) { sim[k] = static_cast<float>(s[k]); sim[8 + k] = static_cast<float>(s[7 + k]); sim[12 + k] = static_cast<float>(s[10 + k]); }
    for (int k = 0; k < 4; ++k) sim[4 + k] = static_cast<float>(s[3 + k]);
    const SimOffsets so(nl);
    const SnapshotOffsets sn(nl);
    for (int j = 0; j < nl; ++j) {
        for (int k = 0; k < 4; ++k) sim[so.jpos + 4 * j + k] = static_cast<float>(s[sn.jpos + 4 * j + k]);
        for (int k = 0; k < M.link[j].ndof; ++k) sim[so.jvel + 4 * j + k] = static_cast<float>(s[sn.jvel + 3 * j + k]);
        for (int c = 0; c < 4; ++c) for (int k = 0; k < 12; ++k) man[j * dmk::kManifoldFloats + c * 12 + k] = static_cast<float>(s[sn.manifold + (j * 4 + c) * 12 + k]);
        const double* o = s + sn.pd + 4 * j; float* t = &sim[so.pd + 4 * j];
        if (M.link[j].jtype == dmk::kJSpherical) {
            Quat cr(M.link[j].child_rot[3], M.link[j].child_rot[0], M.link[j].child_rot[1], M.link[j].child_rot[2]);
            Quat q = cr * Quat(o[0], o[1], o[2], o[3]) * dmh::conj(cr);
            t[0] = static_cast<float>(q.x); t[1] = static_cast<float>(q.y); t[2] = static_cast<float>(q.z); t[3] = static_cast<float>(q.w);
        } else if (M.link[j].jtype == dmk::kJRevolute) t[0] = static_cast<float>(o[0]);
    }
    const double* q = s + sn.clocks;
    tm[dmk::kTKin] = q[0]; tm[dmk::kTOrigin] = q[1]; tm[dmk::kTOrigin + 1] = q[2]; tm[dmk::kTOrigin + 2] = q[3];
    for (int k = 0; k < 4; ++k) tm[dmk::kTOriginRot + k] = q[4 + k];
    tm[dmk::kTCtrl] = q[8]; tm[dmk::kTInitOff] = q[9]; tm[dmk::kTPrevAct] = q[10]; tm[dmk::kTTimer] = q[12]; tm[dmk::kTTimerMax] = q[13];
    fl[dmk::kFNeedAction] = q[11] != 0; fl[dmk::kFDone] = 0; fl[dmk::kFTerminate] = 0; fl[dmk::kFValid] = 1; fl[dmk::kFFallen] = 0;
    DM_CUDA(cudaMemcpy(h->st.sim + static_cast<size_t>(env) * ss, sim.data(), ss * sizeof(float), cudaMemcpyHostToDevice));
    DM_CUDA(cudaMemcpy(h->st.manifold + static_cast<size_t>(env) * nl * dmk::kManifoldFloats, man.data(), man.size() * sizeof(float), cudaMemcpyHostToDevice));
    DM_CUDA(cudaMemcpy(h->st.time + static_cast<size_t>(env) * dmk::kTimeDoubles, tm, sizeof(tm), cudaMemcpyHostToDevice));
    DM_CUDA(cudaMemcpy(h->st.flags + static_cast<size_t>(env) * dmk::kFlagInts, fl, sizeof(fl), cudaMemcpyHostToDevice));
    return 0;
}
// ---- whole-batch state (dm_state_size / dm_save_state / dm_load_state): a header, then the per-environment device blocks in DevState order
namespace {
constexpr char kStateMagic[8] = {'D', 'M', 'S', 'T', 'A', 'T', 'E', 0};
constexpr uint32_t kStateVersion = 1;
struct StateHeader {
    char magic[8];
    uint32_t version, dynamics;   // dynamics: 0 without a randomised dynamics table, else a hash of its bounds (dynamics_hash)
    uint64_t bytes;
    int32_t num_envs, padded_envs, W, links, state_size, action_size, goal_size, amp_obs_size, num_clips;
    int32_t dyn_table;   // 1: the blob ends with a dynamics table (dm_set_dynamics or dm_set_dynamics_randomization); 0: none
    uint64_t seed, env_offset, model;
    char scene[32];
    // host state that changes later results
    uint64_t amp_calls, expert_samples;
    int32_t mode;
    uint32_t push_schedule;   // 0: no push schedule; otherwise a hash of its parameters (push_schedule_hash), whose blocks end the blob
    double time_lim_min, time_lim_max;
};
struct StateBlock { void* dev; size_t bytes; };
// the device blocks of the blob, in order; null blocks of the scene (task, taskx, clip outside the task scenes) are absent
std::vector<StateBlock> state_blocks(const dm_handle* h) {
    const size_t N = static_cast<size_t>(h->padded_envs);
    const auto& M = h->hm;
    const dmk::DevState& s = h->st;
    std::vector<StateBlock> b = {{s.sim, N * dmk::sim_stride(M.nl) * sizeof(float)}, {s.time, N * dmk::kTimeDoubles * sizeof(double)},
                                 {s.flags, N * dmk::kFlagInts * sizeof(int)}, {s.manifold, N * M.nl * dmk::kManifoldFloats * sizeof(float)},
                                 {s.hist, N * 2 * M.pose_dim * sizeof(float)}, {s.task, N * dmk::kTaskDoubles * sizeof(double)},
                                 {s.taskx, N * dmk::kTaskExtDoubles * sizeof(double)}, {s.clip, N * sizeof(int)}, {s.load, N * sizeof(int)}};
    b.erase(std::remove_if(b.begin(), b.end(), [](const StateBlock& x) { return x.dev == nullptr; }), b.end());
    if (h->d_push_sched) {   // a push schedule: its push table and schedule block (manual dm_set_pushes tables are not part of the blob)
        b.push_back({h->d_push, N * sizeof(dmk::DevPush)});
        b.push_back({h->d_push_sched, N * dmk::kPushSchedDoubles * sizeof(double)});
    }
    if (h->d_dyn) b.push_back({h->d_dyn, N * sizeof(dmk::DevDyn)});   // a dynamics table ends the blob
    return b;
}
// the state header's push_schedule field: 0 without a schedule, else FNV-1a over its parameters folded to 32 bits and never 0
uint32_t push_schedule_hash(const dm_handle* h) {
    if (!h->d_push_sched) return 0;
    const unsigned char* p = reinterpret_cast<const unsigned char*>(&h->push_sched);
    uint64_t x = 1469598103934665603ull;
    for (size_t i = 0; i < sizeof(h->push_sched); ++i) { x ^= p[i]; x *= 1099511628211ull; }
    const uint32_t v = static_cast<uint32_t>(x ^ (x >> 32));
    return v ? v : 1u;
}
// the state header's dynamics field: 0 without a randomised table (none, or dm_set_dynamics), else FNV-1a over the bounds, folded, never 0
uint32_t dynamics_hash(const dm_handle* h) {
    if (!h->dyn_random) return 0;
    const unsigned char* p = reinterpret_cast<const unsigned char*>(h->dyn_rand.lohi);
    uint64_t x = 1469598103934665603ull;
    for (size_t i = 0; i < sizeof(h->dyn_rand.lohi); ++i) { x ^= p[i]; x *= 1099511628211ull; }
    const uint32_t v = static_cast<uint32_t>(x ^ (x >> 32));
    return v ? v : 1u;
}
// FNV-1a over the model blob with the fields that change at run time (time limits, mode) cleared: tells handles of different characters,
// controllers or clips apart when every count matches
uint64_t model_hash(const dm_handle* h) {
    dmk::DevModel m;
    std::memcpy(&m, &h->hm, sizeof(m));   // bytewise, padding included (build_device_model clears it)
    m.time_lim_min = m.time_lim_max = 0.0; m.test_mode = 0;
    const unsigned char* p = reinterpret_cast<const unsigned char*>(&m);
    uint64_t x = 1469598103934665603ull;
    for (size_t i = 0; i < sizeof(m); ++i) { x ^= p[i]; x *= 1099511628211ull; }
    return x;
}
StateHeader state_header(const dm_handle* h) {
    StateHeader H;
    std::memset(&H, 0, sizeof(H));
    std::memcpy(H.magic, kStateMagic, sizeof(H.magic));
    H.version = kStateVersion; H.dynamics = dynamics_hash(h); H.dyn_table = h->d_dyn ? 1 : 0;
    H.bytes = sizeof(StateHeader);
    for (const StateBlock& b : state_blocks(h)) H.bytes += b.bytes;
    const auto& M = h->hm;
    H.num_envs = h->num_envs; H.padded_envs = h->padded_envs; H.W = h->W; H.links = M.nl; H.state_size = M.state_size; H.action_size = M.action_size;
    H.goal_size = goal_size(M); H.amp_obs_size = M.amp_obs_size; H.num_clips = h->ctab.num_clips;
    H.seed = h->seed; H.env_offset = h->env_offset; H.model = model_hash(h);
    std::snprintf(H.scene, sizeof(H.scene), "%s", h->sa.cfg.scene.c_str());
    H.amp_calls = h->amp_calls; H.expert_samples = h->expert_samples; H.mode = h->mode; H.push_schedule = push_schedule_hash(h);
    H.time_lim_min = M.time_lim_min; H.time_lim_max = M.time_lim_max;
    return H;
}
}  // namespace

int dm_state_size(dm_handle* h, size_t* bytes) {
    DM_DEVICE(h);
    *bytes = state_header(h).bytes;
    return 0;
}
int dm_save_state(dm_handle* h, void* h_out) {
    DM_DEVICE(h);
    if (h->d_push && !h->d_push_sched) {   // a pending push set by dm_set_pushes is not part of the state blob
        std::vector<int32_t> body(static_cast<size_t>(h->num_envs));
        if (dm_get_pushes(h, body.data())) return 1;
        for (int e = 0; e < h->num_envs; ++e)
            if (body[e] >= 0) { g_err = "dm_save_state: environment " + std::to_string(e) + " has a pending push (dm_set_pushes); the state blob does not carry pushes"; return fail(); }
    }
    const StateHeader H = state_header(h);
    char* o = static_cast<char*>(h_out);
    std::memcpy(o, &H, sizeof(H));
    o += sizeof(H);
    for (const StateBlock& b : state_blocks(h)) {
        DM_CUDA(cudaMemcpyAsync(o, b.dev, b.bytes, cudaMemcpyDeviceToHost, h->stream));
        o += b.bytes;
    }
    DM_CUDA(cudaStreamSynchronize(h->stream));
    return 0;
}
int dm_load_state(dm_handle* h, const void* h_in) {
    DM_DEVICE(h);
    StateHeader in;
    std::memcpy(&in, h_in, sizeof(in));
    const StateHeader mine = state_header(h);
    auto refuse = [](const char* field) { g_err = std::string("dm_load_state: the state was saved by a handle with another ") + field; return fail(); };
    if (std::memcmp(in.magic, kStateMagic, sizeof(in.magic)) != 0) { g_err = "dm_load_state: not a state blob (magic)"; return fail(); }
    if (in.version != kStateVersion) return refuse("layout version");
    if (std::strncmp(in.scene, mine.scene, sizeof(in.scene)) != 0) return refuse("scene");
    if (in.num_envs != mine.num_envs) return refuse("num_envs");
    if (in.padded_envs != mine.padded_envs) return refuse("padded_envs");
    if (in.W != mine.W) return refuse("tile width W");
    if (in.links != mine.links) return refuse("link count");
    if (in.state_size != mine.state_size) return refuse("state size");
    if (in.action_size != mine.action_size) return refuse("action size");
    if (in.goal_size != mine.goal_size) return refuse("goal size");
    if (in.amp_obs_size != mine.amp_obs_size) return refuse("AMP observation size");
    if (in.num_clips != mine.num_clips) return refuse("clip count");
    if (in.seed != mine.seed) return refuse("seed");
    if (in.env_offset != mine.env_offset) return refuse("global env offset");
    if (in.model != mine.model) return refuse("model (character, controller or clips)");
    if (in.push_schedule != mine.push_schedule) return refuse("push schedule (dm_set_push_schedule: none, or other parameters)");
    if (in.dyn_table != mine.dyn_table) return refuse("dynamics table (dm_set_dynamics, dm_set_dynamics_randomization: one, or none)");
    if (in.dynamics != mine.dynamics) return refuse("dynamics randomisation (dm_set_dynamics_randomization: none, or other bounds)");
    if (in.bytes != mine.bytes) return refuse("byte size");
    const char* p = static_cast<const char*>(h_in) + sizeof(in);
    for (const StateBlock& b : state_blocks(h)) {
        DM_CUDA(cudaMemcpyAsync(b.dev, p, b.bytes, cudaMemcpyHostToDevice, h->stream));
        p += b.bytes;
    }
    DM_CUDA(cudaStreamSynchronize(h->stream));
    h->amp_calls = in.amp_calls; h->expert_samples = in.expert_samples;
    h->hm.time_lim_min = in.time_lim_min; h->hm.time_lim_max = in.time_lim_max;
    if (upload_time_limits(h)) return 1;
    return dm_set_mode(h, in.mode);
}

int dm_get_section_profile(dm_handle* h, uint32_t* out, int* num_blocks, int* warps_per_block) {
    DM_DEVICE(h);
    if (!h->st.prof) { g_err = "dm_get_section_profile: this library is not the profile build (make -C deepmimic_b200/csrc profile)"; return fail(); }
    const int blocks = h->padded_envs / h->tiles, warps = h->tiles * h->W / 32;
    if (num_blocks) *num_blocks = blocks;
    if (warps_per_block) *warps_per_block = warps;
    if (out) {
        DM_CUDA(cudaStreamSynchronize(h->stream));
        DM_CUDA(cudaMemcpy(out, h->st.prof, static_cast<size_t>(blocks) * warps * dmk::kProfCounters * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    }
    return 0;
}
int dm_get_counters(dm_handle* h, int64_t* out) {
    DM_DEVICE(h);
    DM_CUDA(cudaStreamSynchronize(h->stream));
    std::vector<int> fl(static_cast<size_t>(h->padded_envs) * dmk::kFlagInts);
    DM_CUDA(cudaMemcpy(fl.data(), h->st.flags, fl.size() * sizeof(int), cudaMemcpyDeviceToHost));
    int64_t over = 0;
    for (int e = 0; e < h->num_envs; ++e) over += fl[static_cast<size_t>(e) * dmk::kFlagInts + dmk::kFRowOverflow];
    out[0] = h->launches; out[1] = over;
    return 0;
}

}  // extern "C"
