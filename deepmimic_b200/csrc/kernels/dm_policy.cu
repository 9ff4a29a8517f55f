// Policy-rate (30 Hz) kernels, one tile of W lanes per environment, lane = link/joint:
//   dm_observe_kernel   : cCtController::RecordState (R/DeepMimicCore/sim/CtController.cpp:281-293,373-478)
//                       + cSceneImitate::CalcReward / CalcRewardImitate (scenes/SceneImitate.cpp:7-127,163-175)
//                         against the mocap frame sampled like cMotion::CalcFrame / cKinTree::LerpPoses
//                         (anim/Motion.cpp:267-293,486-515; anim/KinTree.cpp:1336-1378)
//   dm_set_action_kernel: cCtPDController::ApplyAction -> ConvertActionToTargetPose (sim/CtPDController.cpp:97-166)
//   dm_reset_kernel     : cSceneSimChar::ResetScene chain (SURVEY.md 3d) for the environments whose done flag is set
//   dm_pose_kernel      : cSimCharacter::BuildPose / BuildVel (sim/SimCharacter.cpp:1428-1507) of every environment
#include "dm_model.cuh"

namespace dmk {

namespace {

template <int W>
struct TileP {
    static __device__ __forceinline__ float shfl(float v, int src) { return __shfl_sync(0xffffffffu, v, src, W); }
    static __device__ __forceinline__ int shfli(int v, int src) { return __shfl_sync(0xffffffffu, v, src, W); }
    static __device__ __forceinline__ V3 shfl3(V3 v, int src) { return mk3(shfl(v.x, src), shfl(v.y, src), shfl(v.z, src)); }
    static __device__ __forceinline__ float sum(float v) {
#pragma unroll
        for (int o = W / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o, W);
        return v;
    }
    static __device__ __forceinline__ float minf(float v) {
#pragma unroll
        for (int o = W / 2; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o, W));
        return v;
    }
};

__device__ __forceinline__ float norm_angle(float t) {
    float n = fmodf(t, 6.283185307179586f);
    if (n > 3.14159265358979f) n -= 6.283185307179586f;
    else if (n < -3.14159265358979f) n += 6.283185307179586f;
    return n;
}
// Eigen::Quaternion::slerp (the reference's interpolation, anim/KinTree.cpp:1547,1564)
__device__ __forceinline__ Q4 eigen_slerp(Q4 a, float t, Q4 b) {
    float d = a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w;
    float ad = fabsf(d), s0, s1;
    if (ad >= 1.0f - 1.1920929e-7f) { s0 = 1.0f - t; s1 = t; }
    else { float th = acosf(ad), st = sinf(th); s0 = sinf((1.0f - t) * th) / st; s1 = sinf(t * th) / st; }
    if (d < 0.f) s1 = -s1;
    return mkq(s0 * a.x + s1 * b.x, s0 * a.y + s1 * b.y, s0 * a.z + s1 * b.z, s0 * a.w + s1 * b.w);
}
// squared rotation angle between two unit quaternions with cMathUtil::QuatTheta's dead zone (sin(theta/2) <= 1e-4 -> 0)
__device__ __forceinline__ float quat_theta_sq(Q4 a, Q4 b) {
    Q4 dq = qmul(b, qconj(a));
    float s = sqrtf(dq.x * dq.x + dq.y * dq.y + dq.z * dq.z);
    if (!(s > 0.0001f)) return 0.f;
    float th = 2.0f * atan2f(s, fabsf(dq.w));
    return th * th;
}
// MT: DevModel (the scene's clip) or ClipModel (one clip of a dataset) -- both expose motion_dur / loop_motion / num_frames / pose_dim
template <class MT>
__device__ __forceinline__ void frame_index(const MT& M, const double* ft, double time, int& idx, double& blend, int& cyc) {
    const double dur = M.motion_dur;
    if (!M.loop_motion) {
        cyc = static_cast<int>(floor(time / dur)); cyc = cyc < 0 ? 0 : (cyc > 1 ? 1 : cyc);
        if (time <= 0) { idx = 0; blend = 0; return; }
        if (time >= dur) { idx = M.num_frames - 2; blend = 1; return; }
    } else cyc = static_cast<int>(floor(time / dur));
    double tt = time - cyc * dur;
    int lo = 0, hi = M.num_frames;   // upper_bound(tt) - 1
    while (hi - lo > 1) { int mid = (lo + hi) >> 1; if (ft[mid] <= tt) lo = mid; else hi = mid; }
    if (lo > M.num_frames - 2) lo = M.num_frames - 2;
    idx = lo;
    blend = (tt - ft[lo]) / (ft[lo + 1] - ft[lo]);
}
// mocap sample for joint `lane` in DeepMimic pose layout: returns the joint quaternion (w-first stored in the table) as Q4 xyzw,
// the revolute angle in .x, and the joint velocity
struct KinJoint { Q4 q; V3 w; float ang, angvel; };
__device__ __forceinline__ KinJoint sample_joint(const DevLink& L, const float* f0, const float* f1, const float* v0, const float* v1, float bl, bool is_root) {
    KinJoint k; k.q = mkq(0, 0, 0, 1); k.w = mk3(0, 0, 0); k.ang = 0; k.angvel = 0;
    if (is_root) {
        Q4 a = mkq(f0[4], f0[5], f0[6], f0[3]), b = mkq(f1[4], f1[5], f1[6], f1[3]);
        k.q = qnormalize(eigen_slerp(a, bl, b));
        k.w = mk3((1 - bl) * v0[3] + bl * v1[3], (1 - bl) * v0[4] + bl * v1[4], (1 - bl) * v0[5] + bl * v1[5]);
    } else if (L.jtype == kJSpherical) {
        const int o = L.pose_off;
        Q4 a = mkq(f0[o + 1], f0[o + 2], f0[o + 3], f0[o]), b = mkq(f1[o + 1], f1[o + 2], f1[o + 3], f1[o]);
        k.q = eigen_slerp(a, bl, b);
        k.w = mk3((1 - bl) * v0[o] + bl * v1[o], (1 - bl) * v0[o + 1] + bl * v1[o + 1], (1 - bl) * v0[o + 2] + bl * v1[o + 2]);
    } else if (L.jtype == kJRevolute) {
        const int o = L.pose_off;
        k.ang = (1 - bl) * f0[o] + bl * f1[o];
        k.angvel = (1 - bl) * v0[o] + bl * v1[o];
    }
    return k;
}


// DeepMimic pose / vel entries of one joint from the simulated state: cSimCharacter::BuildPose / BuildVel (SimCharacter.cpp:1428-1507),
// cSimBodyJoint::BuildPose / BuildVel (SimBodyJoint.cpp:342-445).  q: joint rotation (x,y,z,w) in the joint frame (root: world rotation),
// p: root position / (angle, -, -), w: joint-local angular velocity / (rate, -, -), v: root linear velocity.
struct DmJoint { Q4 q; V3 p, w, v; };
__device__ __forceinline__ DmJoint sim_joint_to_dm(const DevModel& M, const DevLink& L, const float* sim, int j, bool is_root) {
    DmJoint d; d.q = mkq(0, 0, 0, 1); d.p = mk3(0, 0, 0); d.w = mk3(0, 0, 0); d.v = mk3(0, 0, 0);
    const float inv_scale = 1.0f / M.scale;
    if (is_root) {
        d.p = inv_scale * mk3(sim[0], sim[1], sim[2]);
        d.q = qconj(mkq(sim[4], sim[5], sim[6], sim[7]));
        if (d.q.w < 0) d.q = mkq(-d.q.x, -d.q.y, -d.q.z, -d.q.w);
        d.w = mk3(sim[8], sim[9], sim[10]);
        d.v = inv_scale * mk3(sim[12], sim[13], sim[14]);
        return d;
    }
    const float4 jp = reinterpret_cast<const float4*>(sim + 16)[j];
    const float4 jv = reinterpret_cast<const float4*>(sim + 16 + 4 * M.nl)[j];
    if (L.jtype == kJSpherical) {
        const Q4 cr = mkq(L.child_rot[0], L.child_rot[1], L.child_rot[2], L.child_rot[3]);
        Q4 q = qmul(qmul(qconj(cr), mkq(jp.x, jp.y, jp.z, jp.w)), cr);
        if (q.w < 0) q = mkq(-q.x, -q.y, -q.z, -q.w);
        d.q = q;
        d.w = qrot(qconj(cr), mk3(jv.x, jv.y, jv.z));
    } else if (L.jtype == kJRevolute) { d.p.x = norm_angle(jp.x); d.w.x = jv.x; }
    return d;
}
// write / read one joint of a DeepMimic pose | vel pair stored as floats (quaternions w-first, like the reference's vectors)
__device__ __forceinline__ void hist_store(float* h, int pose_dim, const DevLink& L, bool is_root, const DmJoint& d) {
    float* p = h + L.pose_off; float* v = h + pose_dim + L.pose_off;
    if (is_root) { p[0] = d.p.x; p[1] = d.p.y; p[2] = d.p.z; p[3] = d.q.w; p[4] = d.q.x; p[5] = d.q.y; p[6] = d.q.z; v[0] = d.v.x; v[1] = d.v.y; v[2] = d.v.z; v[3] = d.w.x; v[4] = d.w.y; v[5] = d.w.z; v[6] = 0.f; }
    else if (L.jtype == kJSpherical) { p[0] = d.q.w; p[1] = d.q.x; p[2] = d.q.y; p[3] = d.q.z; v[0] = d.w.x; v[1] = d.w.y; v[2] = d.w.z; v[3] = 0.f; }
    else if (L.jtype == kJRevolute) { p[0] = d.p.x; v[0] = d.w.x; }
}
__device__ __forceinline__ DmJoint hist_load(const float* h, int pose_dim, const DevLink& L, bool is_root) {
    DmJoint d; d.q = mkq(0, 0, 0, 1); d.p = mk3(0, 0, 0); d.w = mk3(0, 0, 0); d.v = mk3(0, 0, 0);
    const float* p = h + L.pose_off; const float* v = h + pose_dim + L.pose_off;
    if (is_root) { d.p = mk3(p[0], p[1], p[2]); d.q = mkq(p[4], p[5], p[6], p[3]); d.v = mk3(v[0], v[1], v[2]); d.w = mk3(v[3], v[4], v[5]); }
    else if (L.jtype == kJSpherical) { d.q = mkq(p[1], p[2], p[3], p[0]); d.w = mk3(v[0], v[1], v[2]); }
    else if (L.jtype == kJRevolute) { d.p.x = p[0]; d.w.x = v[0]; }
    return d;
}
// raw clip sample (cMotion::CalcFrame / CalcFrameVel: no origin, no cycle offset) for joint `lane`
template <class MT>
__device__ __forceinline__ DmJoint clip_joint(const MT& M, const DevLink& L, const double* ft, const float* frames, const float* frame_vel, double time, bool is_root) {
    int idx, cyc; double bld;
    frame_index(M, ft, time, idx, bld, cyc);
    const float blv = static_cast<float>(bld);
    const float bl = static_cast<float>(fmin(fmax(bld, 0.0), 1.0));
    const float* f0 = frames + static_cast<size_t>(idx) * M.pose_dim; const float* f1 = f0 + M.pose_dim;
    const float* v0 = frame_vel + static_cast<size_t>(idx) * M.pose_dim; const float* v1 = v0 + M.pose_dim;
    const bool over = !M.loop_motion && time >= M.motion_dur;
    KinJoint k = sample_joint(L, f0, f1, v0, v1, bl, is_root);
    DmJoint d; d.q = k.q; d.p = mk3(k.ang, 0, 0); d.w = (L.jtype == kJRevolute && !is_root) ? mk3(0, 0, 0) : mk3(0, 0, 0); d.v = mk3(0, 0, 0);
    const int o = L.pose_off;
    if (is_root) {
        d.p = mk3((1 - bl) * f0[0] + bl * f1[0], (1 - bl) * f0[1] + bl * f1[1], (1 - bl) * f0[2] + bl * f1[2]);
        if (!over) { d.v = mk3((1 - blv) * v0[0] + blv * v1[0], (1 - blv) * v0[1] + blv * v1[1], (1 - blv) * v0[2] + blv * v1[2]);
                     d.w = mk3((1 - blv) * v0[3] + blv * v1[3], (1 - blv) * v0[4] + blv * v1[4], (1 - blv) * v0[5] + blv * v1[5]); }
    } else if (L.jtype == kJSpherical) { if (!over) d.w = mk3((1 - blv) * v0[o] + blv * v1[o], (1 - blv) * v0[o + 1] + blv * v1[o + 1], (1 - blv) * v0[o + 2] + blv * v1[o + 2]); }
    else if (L.jtype == kJRevolute) { if (!over) d.w.x = (1 - blv) * v0[o] + blv * v1[o]; }
    return d;
}
// the clip description a kernel samples from: the model itself, or the per-environment dataset clip in the CLIPS instantiations
template <bool CLIPS> struct ClipPick;
template <> struct ClipPick<false> { static __device__ __forceinline__ const DevModel& get(const DevModel& m, const ClipModel&) { return m; } };
template <> struct ClipPick<true> { static __device__ __forceinline__ const ClipModel& get(const DevModel&, const ClipModel& c) { return c; } };

// The kinematic character at the environment's kin time (cKinCharacter::CalcPose / CalcVel, KinCharacter.cpp:363-406): the clip sample of
// joint `L` (kj; a finished non-looping clip is at rest) and the root in the world -- cycle offset of a looping clip, origin rotation and
// position applied, quaternion with w >= 0.  CLIPS: the environment `clip_env`'s own clip of the dataset.  What dm_observe's imitation reward
// compares against and dm_record_kin_pose writes.
struct KinSample {
    KinJoint kj;
    V3 org, kroot, kroot_v, kroot_w;
    Q4 krootq;
};
template <bool CLIPS>
__device__ __forceinline__ KinSample kin_sample(const DevModel& M, const DevLink& L, const DevState& st, const double* __restrict__ frame_times,
                                                const float* __restrict__ frames, const float* __restrict__ frame_vel, const double* tm, int clip_env,
                                                bool is_root) {
    KinSample s;
    ClipModel CM;
    if constexpr (CLIPS) {
        const ClipInfo& ci = st.ctab->info[st.clip[clip_env]];
        CM = clip_model(ci, M.pose_dim, M.query_dt);
        frame_times += ci.frame_off; frames += static_cast<size_t>(ci.frame_off) * M.pose_dim; frame_vel += static_cast<size_t>(ci.frame_off) * M.pose_dim;
    }
    const auto& KM = ClipPick<CLIPS>::get(M, CM);
    int idx, cyc; double bld;
    frame_index(KM, frame_times, tm[kTKin], idx, bld, cyc);
    bld = fmin(fmax(bld, 0.0), 1.0);
    const float bl = static_cast<float>(bld);
    const float* f0 = frames + static_cast<size_t>(idx) * M.pose_dim; const float* f1 = f0 + M.pose_dim;
    const float* v0 = frame_vel + static_cast<size_t>(idx) * M.pose_dim; const float* v1 = v0 + M.pose_dim;
    const bool clip_over = !KM.loop_motion && tm[kTKin] >= KM.motion_dur;
    s.kj = sample_joint(L, f0, f1, v0, v1, bl, is_root);
    if (clip_over) { s.kj.w = mk3(0, 0, 0); s.kj.angvel = 0; }
    const Q4 orot = mkq(static_cast<float>(tm[kTOriginRot + 1]), static_cast<float>(tm[kTOriginRot + 2]), static_cast<float>(tm[kTOriginRot + 3]), static_cast<float>(tm[kTOriginRot]));
    s.org = mk3(static_cast<float>(tm[kTOrigin]), static_cast<float>(tm[kTOrigin + 1]), static_cast<float>(tm[kTOrigin + 2]));
    // kinematic root in the world
    V3 kroot = mk3((1 - bl) * f0[0] + bl * f1[0] + (KM.loop_motion ? cyc * KM.cycle_delta[0] : 0.f), (1 - bl) * f0[1] + bl * f1[1],
                   (1 - bl) * f0[2] + bl * f1[2] + (KM.loop_motion ? cyc * KM.cycle_delta[2] : 0.f));
    s.kroot = qrot(orot, kroot) + s.org;
    V3 kroot_v = mk3((1 - bl) * v0[0] + bl * v1[0], (1 - bl) * v0[1] + bl * v1[1], (1 - bl) * v0[2] + bl * v1[2]);
    if (clip_over) kroot_v = mk3(0, 0, 0);
    s.kroot_v = qrot(orot, kroot_v);
    {
        KinJoint kr = sample_joint(M.link[0], f0, f1, v0, v1, bl, true);
        s.krootq = qmul(orot, kr.q);
        if (s.krootq.w < 0) s.krootq = mkq(-s.krootq.x, -s.krootq.y, -s.krootq.z, -s.krootq.w);
        s.kroot_w = clip_over ? mk3(0, 0, 0) : qrot(orot, kr.w);
    }
    return s;
}

}  // namespace

// obs: [N x state_size] floats, reward: [N] floats.  Either pointer may be null.
// Outputs go to `fan.n` destinations with identical layout (ObsFan, dm_model.cuh): destination 0 is this GPU's buffer, the others are the
// same slots of the peers' exchange buffers, mapped through CUDA IPC -- the observation rows are staged in shared memory and leave the SM as
// 16-byte stores, so the multi-GPU "all-gather" of the policy step is the store phase of this kernel (NVLink P2P writes), not a collective.
// CLIPS (--kin_ctrl clips, AMP task scenes): the imitation reward is taken against the environment's own active clip of the dataset
// (st.clip / st.ctab) -- BASELINE.json config 5 records it next to the AMP observations and the task reward.
// DYN (dm_observe_dyn_kernel, handles with a dynamics table): the COM velocities of the reward weigh the links by the environment's own masses.
template <int W, int BLOCK, bool CLIPS, bool DYN>
__device__ __forceinline__ void observe_body(const DevModel* __restrict__ gm, DevState st, const double* __restrict__ frame_times,
                                             const float* __restrict__ frames, const float* __restrict__ frame_vel,
                                             ObsFan fan, int num_real_envs, const DevDyn* __restrict__ dyn) {
    using T = TileP<W>;
    extern __shared__ __align__(16) float srow[];   // [tiles x state_size] observation rows of this block
    const bool want_obs = fan.obs[0] != nullptr, want_reward = fan.rew[0] != nullptr;
    const int tiles = BLOCK / W, tile = threadIdx.x / W, lane = threadIdx.x % W;
    const int env = blockIdx.x * tiles + tile;
    const DevModel& M = *gm;
    const int nl = M.nl;
    const bool act = lane < nl;
    const int li = act ? lane : nl - 1;
    const DevLink& L = M.link[li];
    const int ss = sim_stride(nl);
    const float* sim = st.sim + static_cast<size_t>(env) * ss;
    const double* tm = st.time + static_cast<size_t>(env) * kTimeDoubles;
    const int* fl = st.flags + static_cast<size_t>(env) * kFlagInts;
    const float inv_scale = 1.0f / M.scale;
    const V3 basePos = mk3(sim[0], sim[1], sim[2]);
    const Q4 baseQuat = mkq(sim[4], sim[5], sim[6], sim[7]);
    const V3 baseOmega = mk3(sim[8], sim[9], sim[10]), baseVel = mk3(sim[12], sim[13], sim[14]);
    const float4 jp = reinterpret_cast<const float4*>(sim + 16)[li];
    const float4 jv = reinterpret_cast<const float4*>(sim + 16 + 4 * nl)[li];
    const int parent = L.parent, plane = parent >= 0 ? parent : 0, level = act ? L.level : 1000, jtype = L.jtype;
    const V3 dvec = mk3(L.dvec[0], L.dvec[1], L.dvec[2]), evec = mk3(L.evec[0], L.evec[1], L.evec[2]);
    const Q4 zrot = mkq(L.zrot[0], L.zrot[1], L.zrot[2], L.zrot[3]);
    const V3 axis = mk3(L.axis[0], L.axis[1], L.axis[2]);

    // ---- forward kinematics of the simulated character (world->link rotation, COM position, COM twist in the link frame)
    Q4 cached;
    if (jtype == kJSpherical) cached = qmul(mkq(jp.x, jp.y, jp.z, -jp.w), zrot);
    else if (jtype == kJRevolute) { float s, c; sincosf(-0.5f * jp.x, &s, &c); cached = qmul(mkq(axis.x * s, axis.y * s, axis.z * s, c), zrot); }
    else cached = zrot;
    const M3 R = qmat(cached);
    const V3 r = dvec + mul(R, evec);
    const M3 Rwb = qmat(baseQuat);
    M3 Rwl = mul(R, Rwb);
    V3 pos = basePos + mulT(Rwl, r);
    V3 wl = mul(Rwb, baseOmega), vl = mul(Rwb, baseVel);
    { V3 w2 = mul(R, wl); vl = mul(R, vl) - cross(r, w2); wl = w2; }
    V3 wJ = mk3(0, 0, 0), vJ = mk3(0, 0, 0);
    if (jtype == kJSpherical) { wJ = mk3(jv.x, jv.y, jv.z); vJ = cross(wJ, dvec); }
    else if (jtype == kJRevolute) { wJ = jv.x * axis; vJ = cross(wJ, dvec); }
    for (int lv = 1; lv <= M.maxlevel; ++lv) {
        M3 pR; for (int k = 0; k < 9; ++k) pR.m[k] = T::shfl(Rwl.m[k], plane);
        V3 pp = T::shfl3(pos, plane), pw_ = T::shfl3(wl, plane), pv_ = T::shfl3(vl, plane);
        if (level == lv) {
            Rwl = mul(R, pR); pos = pp + mulT(Rwl, r);
            V3 w2 = mul(R, pw_); vl = mul(R, pv_) - cross(r, w2) + vJ; wl = w2 + wJ;
        }
    }
    const V3 lin_w = inv_scale * mulT(Rwl, vl), ang_w = mulT(Rwl, wl);   // cSimBodyLink::mLinVel / mAngVel
    const V3 bpos = inv_scale * pos;                                       // cSimObj::GetPos

    // ---- heading frame of the simulated root (cKinTree::BuildOriginTrans, KinTree.cpp:1651-1664)
    const Q4 rootq = qconj(baseQuat);            // root joint rotation (root attach rotation is identity for the shipped characters)
    const V3 root = inv_scale * basePos;
    V3 hx = qrot(rootq, mk3(1, 0, 0));
    const float heading = atan2f(-hx.z, hx.x);
    float sh, ch; sincosf(-heading, &sh, &ch);
    auto rotH = [&](V3 v) { return mk3(ch * v.x + sh * v.z, v.y, -sh * v.x + ch * v.z); };   // rotation about y by -heading

    if (want_obs && env < num_real_envs && act) {
        float* o = srow + tile * M.state_size;
        const int ph = M.phase_input ? 1 : 0;
        if (lane == 0) {
            if (ph) { double p = fmod(tm[kTCtrl] / M.cycle_period, 1.0); o[0] = static_cast<float>(p < 0 ? 1 + p : p); }
            o[ph] = root.y;   // root height above the (flat, y = 0) ground in the origin frame
        }
        const bool is_root = lane == 0;
        V3 cp = bpos;
        if (!(M.rec_world_root_pos && is_root)) { cp = rotH(mk3(bpos.x - root.x, bpos.y, bpos.z - root.z)); cp.y -= root.y; }
        V3 nrm = mk3(Rwl.m[3], Rwl.m[4], Rwl.m[5]), tan = mk3(Rwl.m[0], Rwl.m[1], Rwl.m[2]);   // link y / x axes in world
        V3 lv_ = lin_w, av_ = ang_w;
        if (!(M.rec_world_root_rot && is_root)) { nrm = rotH(nrm); tan = rotH(tan); lv_ = rotH(lv_); av_ = rotH(av_); }
        float* op = o + ph + 1 + 9 * lane;
        op[0] = cp.x; op[1] = cp.y; op[2] = cp.z; op[3] = nrm.x; op[4] = nrm.y; op[5] = nrm.z; op[6] = tan.x; op[7] = tan.y; op[8] = tan.z;
        float* ov = o + ph + 1 + 9 * nl + 6 * lane;
        ov[0] = lv_.x; ov[1] = lv_.y; ov[2] = lv_.z; ov[3] = av_.x; ov[4] = av_.y; ov[5] = av_.z;
    }
    if (want_obs) {
        // flush the block's rows (consecutive environments = one contiguous range of every destination): scalar head up to the first
        // 16-byte boundary, float4 body, scalar tail; every value is read once from shared memory and stored to all destinations
        __syncthreads();
        const int S = M.state_size;
        const int nreal = min(tiles, num_real_envs - static_cast<int>(blockIdx.x) * tiles);
        const size_t base = static_cast<size_t>(blockIdx.x) * tiles * S;
        const int total = nreal > 0 ? nreal * S : 0;
        const int head = min(total, static_cast<int>((4 - (base & 3)) & 3));
        const int nvec = (total - head) >> 2;
        for (int i = threadIdx.x; i < nvec; i += BLOCK) {
            const float* q = srow + head + 4 * i;
            const float4 v = make_float4(q[0], q[1], q[2], q[3]);
            for (int d = 0; d < fan.n; ++d) reinterpret_cast<float4*>(fan.obs[d] + base + head)[i] = v;
        }
        for (int i = threadIdx.x; i < total; i += BLOCK) {
            if (i >= head && i < head + 4 * nvec) continue;
            const float v = srow[i];
            for (int d = 0; d < fan.n; ++d) fan.obs[d][base + i] = v;
        }
    }
    if (fan.done[0] != nullptr && lane == 0 && env < num_real_envs) {
        const float dn = fl[kFDone] ? 1.f : 0.f;
        for (int d = 0; d < fan.n; ++d) fan.done[d][env] = dn;
    }
    if (!want_reward) return;

    // ---- mocap frame at kin_time
    const KinSample ks = kin_sample<CLIPS>(M, L, st, frame_times, frames, frame_vel, tm, env < num_real_envs ? env : 0, lane == 0);
    const KinJoint kj = ks.kj;
    const V3 org = ks.org, kroot = ks.kroot, kroot_v = ks.kroot_v, kroot_w = ks.kroot_w;
    const Q4 krootq = ks.krootq;
    // ---- kinematic FK in the world: joint frames (DeepMimic tree), joint origin position, twist
    const Q4 attq = mkq(L.child_rot[0], L.child_rot[1], L.child_rot[2], L.child_rot[3]);   // joint -> body
    const V3 att_pt = mk3(L.att_pt[0], L.att_pt[1], L.att_pt[2]);
    const Q4 att_rot = mkq(L.att_rot[0], L.att_rot[1], L.att_rot[2], L.att_rot[3]);
    Q4 jq_local = (jtype == kJSpherical) ? kj.q : ((jtype == kJRevolute) ? mkq(0.f, 0.f, sinf(0.5f * kj.ang), cosf(0.5f * kj.ang)) : mkq(0, 0, 0, 1));
    V3 jw_local = (jtype == kJSpherical) ? kj.w : ((jtype == kJRevolute) ? mk3(0.f, 0.f, kj.angvel) : mk3(0, 0, 0));
    Q4 kq = krootq; V3 kp = kroot, kw = kroot_w, kv = kroot_v;   // lane 0 values; other lanes filled level by level
    for (int lv = 1; lv <= M.maxlevel; ++lv) {
        Q4 pq = mkq(T::shfl(kq.x, plane), T::shfl(kq.y, plane), T::shfl(kq.z, plane), T::shfl(kq.w, plane));
        V3 pp = T::shfl3(kp, plane), pw_ = T::shfl3(kw, plane), pv_ = T::shfl3(kv, plane);
        if (level == lv) {
            V3 off = qrot(pq, att_pt);
            kp = pp + off;
            kq = qmul(qmul(pq, att_rot), jq_local);
            kv = pv_ + cross(pw_, off);
            kw = pw_ + qrot(kq, jw_local);
        }
    }
    const V3 body_att = mk3(L.body_att[0], L.body_att[1], L.body_att[2]);
    const V3 kcom_v = kv + cross(kw, qrot(kq, body_att));

    // ---- error terms
    float pose_e = 0.f, vel_e = 0.f, ee_e = 0.f;
    if (act && lane > 0) {
        if (jtype == kJSpherical) {
            Q4 kb = qmul(qmul(attq, kj.q), qconj(attq));            // clip rotation expressed in the body-frame convention of the sim state
            pose_e = quat_theta_sq(mkq(jp.x, jp.y, jp.z, jp.w), kb);
            V3 d = qrot(attq, kj.w) - mk3(jv.x, jv.y, jv.z);
            vel_e = dot(d, d);
        } else if (jtype == kJRevolute) {
            float d = kj.ang - norm_angle(jp.x); pose_e = d * d;
            float dv = kj.angvel - jv.x; vel_e = dv * dv;
        }
        if (L.end_eff) {
            // joint origin of the simulated link: COM + R_lw * child_pos (cSimBodyJoint::CalcWorldPos)
            V3 p0 = bpos + mulT(Rwl, mk3(L.child_pos[0], L.child_pos[1], L.child_pos[2]));
            V3 rel0 = mk3(p0.x - root.x, p0.y, p0.z - root.z);
            V3 rel1 = mk3(kp.x - kroot.x, kp.y - org.y, kp.z - kroot.z);
            rel0 = rotH(rel0);
            V3 khx = qrot(krootq, mk3(1, 0, 0));
            float kh = atan2f(-khx.z, khx.x), s2, c2; sincosf(-kh, &s2, &c2);
            rel1 = mk3(c2 * rel1.x + s2 * rel1.z, rel1.y, -s2 * rel1.x + c2 * rel1.z);
            V3 d = rel1 - rel0;
            ee_e = dot(d, d);
        }
        pose_e *= L.joint_w; vel_e *= L.joint_w;
    }
    if (lane == 0) {
        pose_e = M.link[0].joint_w * quat_theta_sq(rootq, krootq);
        V3 d = kroot_w - baseOmega;
        vel_e = M.link[0].joint_w * dot(d, d);
    }
    const float pose_err = T::sum(act ? pose_e : 0.f), vel_err = T::sum(act ? vel_e : 0.f), end_eff_err = T::sum(act ? ee_e : 0.f);
    float mfrac;
    if constexpr (DYN) { const float* df = dyn[env].f; mfrac = act ? (L.mass * df[kDMass + li]) / df[kDTotalMass] : 0.f; }
    else mfrac = act ? L.mass / M.total_mass : 0.f;
    const V3 com_v0 = mk3(T::sum(mfrac * lin_w.x), T::sum(mfrac * lin_w.y), T::sum(mfrac * lin_w.z));
    const V3 com_v1 = mk3(T::sum(mfrac * kcom_v.x), T::sum(mfrac * kcom_v.y), T::sum(mfrac * kcom_v.z));
    if (lane == 0 && env < num_real_envs) {
        V3 rp0 = root, rp1 = mk3(kroot.x, kroot.y - org.y, kroot.z);
        V3 dp = rp0 - rp1;
        float root_rot_err = quat_theta_sq(rootq, krootq);
        V3 dv = kroot_v - inv_scale * baseVel, dw = kroot_w - baseOmega;
        float root_err = dot(dp, dp) + 0.1f * root_rot_err + 0.01f * dot(dv, dv) + 0.001f * dot(dw, dw);
        V3 dc = com_v1 - com_v0;
        float com_err = 0.1f * dot(dc, dc);
        const float pose_scale = 2.0f / 15 * nl, vel_scale = 0.1f / 15 * nl;
        float rwd = 0.5f * expf(-pose_scale * pose_err) + 0.05f * expf(-vel_scale * vel_err) + 0.15f * expf(-10.f * end_eff_err) +
                    0.2f * expf(-5.f * root_err) + 0.1f * expf(-10.f * com_err);
        if (fl[kFFallen]) rwd = 0.f;
        for (int d = 0; d < fan.n; ++d) fan.rew[d][env] = rwd;
    }
}
template <int W, int BLOCK, bool CLIPS>
__global__ void __launch_bounds__(BLOCK) dm_observe_kernel(const DevModel* __restrict__ gm, DevState st, const double* __restrict__ frame_times,
                                                            const float* __restrict__ frames, const float* __restrict__ frame_vel,
                                                            ObsFan fan, int num_real_envs) {
    observe_body<W, BLOCK, CLIPS, false>(gm, st, frame_times, frames, frame_vel, fan, num_real_envs, nullptr);
}
template <int W, int BLOCK, bool CLIPS>
__global__ void __launch_bounds__(BLOCK) dm_observe_dyn_kernel(const DevModel* __restrict__ gm, DevState st, const double* __restrict__ frame_times,
                                                                const float* __restrict__ frames, const float* __restrict__ frame_vel,
                                                                ObsFan fan, int num_real_envs, const DevDyn* dyn) {
    observe_body<W, BLOCK, CLIPS, true>(gm, st, frame_times, frames, frame_vel, fan, num_real_envs, dyn);
}

namespace {

// seed salts of the expert sampler's two draws ("ampclip", "amptime"): streams of their own, apart from the reset, task and host expert draws
constexpr unsigned long long kExpertClipSalt = 0x616d70636c6970ull, kExpertTimeSalt = 0x616d7074696d65ull;

// AMP observations (cSceneImitateAMP::BuildAMPObs, SceneImitateAMP.cpp:279-397): [pose now | pose prev | vel now | vel prev], one tile per
// row, lane = joint.  expert == 0: "now" is the simulated character, "prev" the history block (RecordAMPObsAgent, :101-113);
// expert != 0: the raw clip at expert_time[env] and one query period earlier, ground height = the kinematic origin's y (:115-140).
// TASKV: the expert sample comes from clip expert_clip[env] of the dataset (cSceneImitateAMP::SampleExpertMotion with a clips controller,
// SceneImitateAMP.cpp:260-277) instead of the scene's single clip.
// SAMPLE (expert != 0): tile `env` is output row `env` of num_real_envs rows and makes its own draws: the clip from the dataset's CDF (TASKV),
// the time from U(0, clip duration), on the counter stream task_u01(seed ^ salt, row, call); the ground height is environment
// row % st.num_real's.  clip_out / time_out (may be null) receive the draws.
template <int W, int BLOCK, bool TASKV, bool SAMPLE>
__device__ __forceinline__ void amp_obs_tile(const DevModel* __restrict__ gm, DevState st, const double* __restrict__ frame_times,
                                             const float* __restrict__ frames, const float* __restrict__ frame_vel, float* __restrict__ out,
                                             int expert, const double* __restrict__ expert_time, int num_real_envs,
                                             const int* __restrict__ expert_clip, unsigned long long seed, unsigned long long call,
                                             int* __restrict__ clip_out, double* __restrict__ time_out) {
    using T = TileP<W>;
    const int tiles = BLOCK / W, tile = threadIdx.x / W, lane = threadIdx.x % W;
    const int env = blockIdx.x * tiles + tile;
    const DevModel& M = *gm;
    const int nl = M.nl;
    const bool act = lane < nl;
    const int li = act ? lane : nl - 1;
    const DevLink& L = M.link[li];
    const int parent = L.parent, plane = parent >= 0 ? parent : 0, level = act ? L.level : 1000, jtype = L.jtype;
    const bool is_root = lane == 0;
    const float* sim = st.sim + static_cast<size_t>(env) * sim_stride(nl);
    const double* tm = st.time + static_cast<size_t>(SAMPLE ? (env < num_real_envs ? env : num_real_envs - 1) % st.num_real : env) * kTimeDoubles;
    DmJoint now, prev;
    float ground_h = 0.f;
    if (!expert) {
        now = sim_joint_to_dm(M, L, sim, li, is_root);
        prev = hist_load(st.hist + static_cast<size_t>(env) * 2 * M.pose_dim, M.pose_dim, L, is_root);
    } else {
        int clip = 0;
        double t;
        if constexpr (SAMPLE) {   // a tail tile (env >= rows) repeats the last row's draws and writes nothing
            const unsigned long long row = env < num_real_envs ? env : num_real_envs - 1;
            double dur = M.motion_dur;
            if constexpr (TASKV) { clip = select_clip(*st.ctab, task_u01(seed ^ kExpertClipSalt, row, call)); dur = st.ctab->info[clip].dur; }
            t = dur * task_u01(seed ^ kExpertTimeSalt, row, call);
            if (lane == 0 && env < num_real_envs) {
                if (clip_out) clip_out[env] = clip;
                if (time_out) time_out[env] = t;
            }
        } else t = expert_time[env];
        ClipModel CM;
        if constexpr (TASKV) {
            const ClipInfo& ci = st.ctab->info[SAMPLE ? clip : expert_clip[env]];
            CM = clip_model(ci, M.pose_dim, M.query_dt);
            frame_times += ci.frame_off; frames += static_cast<size_t>(ci.frame_off) * M.pose_dim; frame_vel += static_cast<size_t>(ci.frame_off) * M.pose_dim;
        }
        const auto& KM = ClipPick<TASKV>::get(M, CM);
        now = clip_joint(KM, L, frame_times, frames, frame_vel, t, is_root);
        prev = clip_joint(KM, L, frame_times, frames, frame_vel, t - M.query_dt, is_root);
        ground_h = static_cast<float>(tm[kTOrigin + 1]);
    }
    // heading of the current root (cKinTree::CalcHeadingRot, KinTree.cpp:1629-1635): rotation about y by -heading
    const Q4 rq_now = mkq(T::shfl(now.q.x, 0), T::shfl(now.q.y, 0), T::shfl(now.q.z, 0), T::shfl(now.q.w, 0));
    const V3 hx = qrot(rq_now, mk3(1, 0, 0));
    const float heading = atan2f(-hx.z, hx.x);
    float sh, ch; sincosf(-heading, &sh, &ch);
    auto rotH = [&](V3 v) { return mk3(ch * v.x + sh * v.z, v.y, -sh * v.x + ch * v.z); };
    const Q4 refq = mkq(0.f, sinf(-0.5f * heading), 0.f, cosf(-0.5f * heading));
    // layout offsets: joint block sizes by an exclusive scan over the lanes
    const int jsz = (!act || is_root) ? 0 : (jtype == kJSpherical ? 6 : (jtype == kJRevolute ? 1 : 0));
    int incl = jsz, eincl = (act && L.end_eff) ? 1 : 0;
#pragma unroll
    for (int o = 1; o < W; o <<= 1) { int t1 = __shfl_up_sync(0xffffffffu, incl, o, W), t2 = __shfl_up_sync(0xffffffffu, eincl, o, W); if (lane >= o) { incl += t1; eincl += t2; } }
    const int joff = incl - jsz, eidx = eincl - ((act && L.end_eff) ? 1 : 0);
    const int jtot = __shfl_sync(0xffffffffu, incl, W - 1, W), etot = __shfl_sync(0xffffffffu, eincl, W - 1, W);
    const int pose_size = 1 + 6 + jtot + 3 * etot;
    const int vel_size = 6 + (M.pose_dim - 7);
    float* o = (env < num_real_envs) ? out + static_cast<size_t>(env) * (2 * (pose_size + vel_size)) : nullptr;
    // kinematic tree of both poses: joint world rotation / origin (cKinTree::JointWorldTrans)
    const V3 att_pt = mk3(L.att_pt[0], L.att_pt[1], L.att_pt[2]);
    const Q4 att_rot = mkq(L.att_rot[0], L.att_rot[1], L.att_rot[2], L.att_rot[3]);
    const V3 body_att = mk3(L.body_att[0], L.body_att[1], L.body_att[2]);
#pragma unroll
    for (int blk = 0; blk < 2; ++blk) {
        const DmJoint& d = blk == 0 ? now : prev;
        Q4 jq = (jtype == kJSpherical) ? d.q : ((jtype == kJRevolute) ? mkq(0.f, 0.f, sinf(0.5f * d.p.x), cosf(0.5f * d.p.x)) : mkq(0, 0, 0, 1));
        Q4 kq = d.q; V3 kp = d.p;       // lane 0: root rotation / position
        for (int lv = 1; lv <= M.maxlevel; ++lv) {
            Q4 pq = mkq(T::shfl(kq.x, plane), T::shfl(kq.y, plane), T::shfl(kq.z, plane), T::shfl(kq.w, plane));
            V3 pp = T::shfl3(kp, plane);
            if (level == lv) { kp = pp + qrot(pq, att_pt); kq = qmul(qmul(pq, att_rot), jq); }
        }
        const V3 root_pos = T::shfl3(kp, 0);
        if (o == nullptr || !act) continue;
        float* ob = o + blk * pose_size;
        if (is_root) {
            ob[0] = d.p.y - ground_h;
            Q4 rr = d.q;
            if (M.amp_local_root) rr = qmul(refq, rr);
            const V3 nrm = qrot(rr, mk3(0, 1, 0)), tan = qrot(rr, mk3(1, 0, 0));   // cMathUtil::CalcNormalTangent (MathUtil.cpp:617-623)
            ob[1] = nrm.x; ob[2] = nrm.y; ob[3] = nrm.z; ob[4] = tan.x; ob[5] = tan.y; ob[6] = tan.z;
        } else if (jtype == kJSpherical) {
            const V3 nrm = qrot(d.q, mk3(0, 1, 0)), tan = qrot(d.q, mk3(1, 0, 0));
            float* q = ob + 7 + joff;
            q[0] = nrm.x; q[1] = nrm.y; q[2] = nrm.z; q[3] = tan.x; q[4] = tan.y; q[5] = tan.z;
        } else if (jtype == kJRevolute) ob[7 + joff] = d.p.x;
        if (L.end_eff) {   // cKinTree::CalcBodyPartPos (KinTree.cpp:272-281) relative to the root, in the heading frame of the current pose
            const V3 bp = rotH(kp + qrot(kq, body_att) - root_pos);
            float* e = ob + 7 + jtot + 3 * eidx;
            e[0] = bp.x; e[1] = bp.y; e[2] = bp.z;
        }
        // velocities (RecordAMPObsVel, :367-397): root lin / ang, then the joint part of the vel vector
        float* ov = o + 2 * pose_size + blk * vel_size;
        if (is_root) {
            V3 rv = d.v, rw = d.w;
            if (M.amp_local_root) { rv = rotH(rv); rw = rotH(rw); }
            ov[0] = rv.x; ov[1] = rv.y; ov[2] = rv.z; ov[3] = rw.x; ov[4] = rw.y; ov[5] = rw.z;
        } else if (jtype == kJSpherical) { float* q = ov + 6 + (L.pose_off - 7); q[0] = d.w.x; q[1] = d.w.y; q[2] = d.w.z; q[3] = 0.f; }
        else if (jtype == kJRevolute) ov[6 + (L.pose_off - 7)] = d.w.x;
    }
}

}  // namespace

template <int W, int BLOCK, bool TASKV>
__global__ void __launch_bounds__(BLOCK) dm_amp_obs_kernel(const DevModel* __restrict__ gm, DevState st, const double* __restrict__ frame_times,
                                                            const float* __restrict__ frames, const float* __restrict__ frame_vel, float* __restrict__ out,
                                                            int expert, const double* __restrict__ expert_time, int num_real_envs,
                                                            const int* __restrict__ expert_clip) {
    amp_obs_tile<W, BLOCK, TASKV, false>(gm, st, frame_times, frames, frame_vel, out, expert, expert_time, num_real_envs, expert_clip, 0, 0, nullptr, nullptr);
}

// `rows` expert AMP observations with their clip and time drawn on the device (amp_obs_tile's SAMPLE): the expert branch of dm_amp_obs_kernel,
// one tile per row.  No host draw, no host synchronisation.
template <int W, int BLOCK, bool TASKV>
__global__ void __launch_bounds__(BLOCK) dm_amp_expert_sample_kernel(const DevModel* __restrict__ gm, DevState st, const double* __restrict__ frame_times,
                                                                      const float* __restrict__ frames, const float* __restrict__ frame_vel,
                                                                      float* __restrict__ out, int rows, unsigned long long seed, unsigned long long call,
                                                                      int* __restrict__ clip_out, double* __restrict__ time_out) {
    amp_obs_tile<W, BLOCK, TASKV, true>(gm, st, frame_times, frames, frame_vel, out, 1, nullptr, rows, nullptr, seed, call, clip_out, time_out);
}

// actions: [N x action_size] floats (DeepMimic action layout)
// LAT (dm_set_action_latency_kernel, handles with a latency table): an environment with a delay d > 0 gets the targets in its pending slot, due at
// the update counter + d (dm_latency.cuh), replacing any action still pending; d = 0 writes the target slot and drops a pending action.  The
// AMP history stays at the action's time.
template <bool LAT>
__device__ __forceinline__ void set_action_body(const DevModel* __restrict__ gm, DevState st, const float* __restrict__ actions, int num_real_envs, DevLat* lat) {
    const DevModel& M = *gm;
    const int gid = blockIdx.x * blockDim.x + threadIdx.x;
    const int env = gid / M.nl, j = gid % M.nl;
    if (env >= num_real_envs) return;
    const DevLink& L = M.link[j];
    // cSceneImitateAMP::UpdateHist (SceneImitateAMP.cpp:167-172): the pose / vel the new action was chosen from
    if (st.hist) hist_store(st.hist + static_cast<size_t>(env) * 2 * M.pose_dim, M.pose_dim, L, j == 0, sim_joint_to_dm(M, L, st.sim + static_cast<size_t>(env) * sim_stride(M.nl), j, j == 0));
    if (j == 0) {
        if constexpr (LAT) {
            const int d = lat[env].delay;
            lat[env].due = d > 0 ? st.flags[static_cast<size_t>(env) * kFlagInts + kFUpdates] + d : -1;
        }
        return;
    }
    const float* a = actions + static_cast<size_t>(env) * M.action_size + L.act_off;
    float4* tgt = reinterpret_cast<float4*>(st.sim + static_cast<size_t>(env) * sim_stride(M.nl) + 16 + 8 * M.nl) + j;
    if constexpr (LAT) {
        if (lat[env].delay > 0) tgt = reinterpret_cast<float4*>(lat[env].tg) + j;
    }
    if (L.jtype == kJSpherical) {
        V3 em = mk3(a[0], a[1], a[2]);
        float len = sqrtf(dot(em, em));
        const float max_len = 6.283185307179586f;
        if (len > max_len) { em = em * (max_len / len); len = max_len; }
        Q4 q = mkq(0, 0, 0, 1);
        if (len > 0.000001f) {
            V3 ax = em * (1.0f / len);
            float th = norm_angle(len), s, c;
            sincosf(0.5f * th, &s, &c);
            q = mkq(ax.x * s, ax.y * s, ax.z * s, c);
        }
        q = qnormalize(q);
        Q4 cr = mkq(L.child_rot[0], L.child_rot[1], L.child_rot[2], L.child_rot[3]);
        q = qmul(qmul(cr, q), qconj(cr));
        *tgt = make_float4(q.x, q.y, q.z, q.w);
    } else if (L.jtype == kJRevolute) {
        *tgt = make_float4(a[0], 0.f, 0.f, 0.f);
    }
}
__global__ void dm_set_action_kernel(const DevModel* __restrict__ gm, DevState st, const float* __restrict__ actions, int num_real_envs) {
    set_action_body<false>(gm, st, actions, num_real_envs, nullptr);
}
__global__ void dm_set_action_latency_kernel(const DevModel* __restrict__ gm, DevState st, const float* __restrict__ actions, int num_real_envs, DevLat* lat) {
    set_action_body<true>(gm, st, actions, num_real_envs, lat);
}

// pose / vel: [num_real_envs x pose_dim] floats, the simulated character in DeepMimic layout (cSimCharacter::BuildPose / BuildVel); either may be
// null.  Block b holds environments [b kPoseEnvsPerBlock, (b + 1) kPoseEnvsPerBlock), one thread per (environment, joint): the AMP history's
// conversion and write rule put each environment's pose | vel pair into shared memory, and the block then stores its pose rows and its vel rows
// as two contiguous ranges.  Padding environments are not written.
__global__ void dm_pose_kernel(const DevModel* __restrict__ gm, DevState st, float* __restrict__ pose, float* __restrict__ vel, int num_real_envs) {
    extern __shared__ float spv[];   // [kPoseEnvsPerBlock x 2 pose_dim]
    const DevModel& M = *gm;
    const int P = M.pose_dim, env0 = blockIdx.x * kPoseEnvsPerBlock;
    const int e = threadIdx.x / M.nl, j = threadIdx.x % M.nl;
    if (e < kPoseEnvsPerBlock && env0 + e < num_real_envs) {
        const DevLink& L = M.link[j];
        hist_store(spv + 2 * P * e, P, L, j == 0, sim_joint_to_dm(M, L, st.sim + static_cast<size_t>(env0 + e) * sim_stride(M.nl), j, j == 0));
    }
    __syncthreads();
    const int n = min(kPoseEnvsPerBlock, num_real_envs - env0) * P;
    const size_t base = static_cast<size_t>(env0) * P;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const float* s = spv + 2 * P * (i / P) + i % P;
        if (pose) pose[base + i] = s[0];
        if (vel) vel[base + i] = s[P];
    }
}

// pose: [num_real_envs x pose_dim] floats, the kinematic character of every environment (kin_sample: cKinCharacter's pose in the world) in
// dm_pose_kernel's layout, quaternions with w >= 0.  One thread per (environment, joint); padding environments are not written.
template <bool CLIPS>
__global__ void dm_kin_pose_kernel(const DevModel* __restrict__ gm, DevState st, const double* __restrict__ frame_times, const float* __restrict__ frames,
                                   const float* __restrict__ frame_vel, float* __restrict__ pose, int num_real_envs) {
    const DevModel& M = *gm;
    const int gid = blockIdx.x * blockDim.x + threadIdx.x;
    const int env = gid / M.nl, j = gid % M.nl;
    if (env >= num_real_envs) return;
    const DevLink& L = M.link[j];
    const KinSample ks = kin_sample<CLIPS>(M, L, st, frame_times, frames, frame_vel, st.time + static_cast<size_t>(env) * kTimeDoubles, env, j == 0);
    float* p = pose + static_cast<size_t>(env) * M.pose_dim + L.pose_off;
    if (j == 0) {
        p[0] = ks.kroot.x; p[1] = ks.kroot.y; p[2] = ks.kroot.z;
        p[3] = ks.krootq.w; p[4] = ks.krootq.x; p[5] = ks.krootq.y; p[6] = ks.krootq.z;
    } else if (L.jtype == kJSpherical) {
        const Q4 q = ks.kj.q.w < 0 ? mkq(-ks.kj.q.x, -ks.kj.q.y, -ks.kj.q.z, -ks.kj.q.w) : ks.kj.q;
        p[0] = q.w; p[1] = q.x; p[2] = q.y; p[3] = q.z;
    } else if (L.jtype == kJRevolute) p[0] = ks.kj.ang;
}
const KinPoseKernel kKinPoseKernels[2] = {dm_kin_pose_kernel<false>, dm_kin_pose_kernel<true>};

// Resets every environment whose done flag is set (or all when force != 0).  kin_time_in / max_time_in (may be null) inject the
// random draws of the reference's reset (CalcRandKinResetTime, cTimer::Reset) so tests can bypass the RNG.
// TASKV (AMP task scenes): every environment samples its own clip of the dataset (st.clip / st.ctab; clip_in injects the controller's draw)
// and the action history is NOT re-initialised (cSceneTargetAMP::Reset bypasses cSceneImitateAMP::Reset, SceneTargetAMP.cpp:129-134).
template <int W, int BLOCK, bool TASKV>
__global__ void __launch_bounds__(BLOCK) dm_reset_kernel(const DevModel* __restrict__ gm, DevState st, const double* __restrict__ frame_times,
                                                          const float* __restrict__ frames, const float* __restrict__ frame_vel, int force,
                                                          const double* __restrict__ kin_time_in, const double* __restrict__ max_time_in,
                                                          const double* __restrict__ rot_theta_in, unsigned long long seed,
                                                          unsigned long long env_id_base, int test_mode, const int* __restrict__ clip_in) {
    using T = TileP<W>;
    const int tiles = BLOCK / W, tile = threadIdx.x / W, lane = threadIdx.x % W;
    const int env = blockIdx.x * tiles + tile;
    const DevModel& M = *gm;
    const int nl = M.nl;
    const bool act = lane < nl;
    const int li = act ? lane : nl - 1;
    const DevLink& L = M.link[li];
    const int ss = sim_stride(nl);
    float* sim = st.sim + static_cast<size_t>(env) * ss;
    double* tm = st.time + static_cast<size_t>(env) * kTimeDoubles;
    int* fl = st.flags + static_cast<size_t>(env) * kFlagInts;
    const bool doit = (force || fl[kFDone] != 0) && env < st.num_real;   // padding environments stay frozen (done) for the life of the handle
    // draws
    const unsigned long long gid = env_id_base + env, cnt = static_cast<unsigned long long>(fl[7]);
    ClipModel CM;
    double reset_time_span = M.motion_dur;
    int new_clip = 0;
    bool recovery = false;   // TASKV, get-up scene: this reset is a recovery episode (decided below, applied at the commit)
    if constexpr (TASKV) {
        const ClipTable& CT = *st.ctab;
        const int prev_clip = st.clip[env];
        // cSceneImitate::ResetKinChar draws the start time from U(0, duration of the clip that was active BEFORE the controller's reset picks
        // the new one) -- CalcRandKinResetTime runs first (SceneImitate.cpp:331-338)
        reset_time_span = CT.info[prev_clip].dur;
        new_clip = doit ? (clip_in ? clip_in[env] : select_clip(CT, task_u01(seed ^ 0x636c697073ull, gid, cnt))) : prev_clip;
        const ClipInfo& ci = CT.info[new_clip];
        CM = clip_model(ci, M.pose_dim, M.query_dt);
        frame_times += ci.frame_off; frames += static_cast<size_t>(ci.frame_off) * M.pose_dim; frame_vel += static_cast<size_t>(ci.frame_off) * M.pose_dim;
    }
    const auto& KM = ClipPick<TASKV>::get(M, CM);
    double kt = kin_time_in ? kin_time_in[env] : task_u01(seed, gid, 3 * cnt) * reset_time_span;
    double mt = max_time_in ? max_time_in[env] : (M.time_lim_min + task_u01(seed, gid, 3 * cnt + 1) * (M.time_lim_max - M.time_lim_min));
    double th = rot_theta_in ? rot_theta_in[env] : (M.rand_rot_reset ? (-3.14159265358979323846 + task_u01(seed, gid, 3 * cnt + 2) * 6.283185307179586) : 0.0);
    if (!M.rand_rot_reset) th = 0.0;
    if (test_mode) mt = M.time_end_lim_max;
    if constexpr (TASKV) {
        // cSceneHeadingAMPGetup::Reset (SceneHeadingAMPGetup.cpp:111-123): after a failed episode a coin decides on a recovery episode -- the fallen
        // character stays as it is, only the scene timer and the controller clocks restart (ResetRecoveryEpisode, :40-58)
        if (M.task_kind == kTaskHeadingGetup) {
            int rec = 0;
            if (lane == 0 && doit) {
                TaskRng rng{M.task_seed, gid, st.task + static_cast<size_t>(env) * kTaskDoubles + kKCounter};
                rec = getup_try_recovery(M.taskx, rng, test_mode != 0, fl[kFTerminate]) ? 1 : 0;
            }
            recovery = T::shfli(rec, 0) != 0;
        }
    }
    int idx, cyc; double bld;
    frame_index(KM, frame_times, kt, idx, bld, cyc);
    bld = fmin(fmax(bld, 0.0), 1.0);
    const float bl = static_cast<float>(bld);
    const float* f0 = frames + static_cast<size_t>(idx) * M.pose_dim; const float* f1 = f0 + M.pose_dim;
    const float* v0 = frame_vel + static_cast<size_t>(idx) * M.pose_dim; const float* v1 = v0 + M.pose_dim;
    // a non-looping clip at or past its end is at rest (cMotion::CalcFrameVel; clip_joint and the observe kernel apply the same rule): a task
    // scene draws the start time from the previous clip's duration, which can lie past the end of a shorter new clip
    const bool clip_over = !KM.loop_motion && kt >= KM.motion_dur;
    KinJoint kj = sample_joint(L, f0, f1, v0, v1, bl, lane == 0);
    if (clip_over) { kj.w = mk3(0, 0, 0); kj.angvel = 0; }
    const float sth = sinf(0.5f * static_cast<float>(th)), cth = cosf(0.5f * static_cast<float>(th));
    const Q4 orot = mkq(0.f, sth, 0.f, cth);
    // root
    V3 rp = mk3((1 - bl) * f0[0] + bl * f1[0] + (KM.loop_motion ? cyc * KM.cycle_delta[0] : 0.f), (1 - bl) * f0[1] + bl * f1[1],
                (1 - bl) * f0[2] + bl * f1[2] + (KM.loop_motion ? cyc * KM.cycle_delta[2] : 0.f));
    V3 rv = mk3((1 - bl) * v0[0] + bl * v1[0], (1 - bl) * v0[1] + bl * v1[1], (1 - bl) * v0[2] + bl * v1[2]);
    KinJoint kr = sample_joint(M.link[0], f0, f1, v0, v1, bl, true);
    if (clip_over) { rv = mk3(0, 0, 0); kr.w = mk3(0, 0, 0); }
    Q4 rq = qmul(orot, kr.q); if (rq.w < 0) rq = mkq(-rq.x, -rq.y, -rq.z, -rq.w);
    rq = qnormalize(rq);
    V3 rw = qrot(orot, kr.w);
    rv = qrot(orot, rv);
    // simulated state := kinematic state, root x,z := 0 (SyncCharacters + SetCharRandPlacement)
    V3 basePos = mk3(0.f, M.scale * rp.y, 0.f);
    Q4 baseQuat = qconj(rq);
    V3 baseVel = M.scale * rv, baseOmega = rw;
    float4 jp = make_float4(0, 0, 0, 1), jv = make_float4(0, 0, 0, 0);
    const Q4 cr = mkq(L.child_rot[0], L.child_rot[1], L.child_rot[2], L.child_rot[3]);
    if (L.jtype == kJSpherical) {
        Q4 q = qmul(qmul(cr, kj.q), qconj(cr));
        V3 w = qrot(cr, kj.w);
        jp = make_float4(q.x, q.y, q.z, q.w); jv = make_float4(w.x, w.y, w.z, 0.f);
    } else if (L.jtype == kJRevolute) { jp = make_float4(kj.ang, 0, 0, 0); jv = make_float4(kj.angvel, 0, 0, 0); }
    // ---- FK for cSceneSimChar::ResolveCharGroundIntersect: lowest AABB point of every link shape
    const int parent = L.parent, plane = parent >= 0 ? parent : 0, level = act ? L.level : 1000, jtype = L.jtype;
    const V3 dvec = mk3(L.dvec[0], L.dvec[1], L.dvec[2]), evec = mk3(L.evec[0], L.evec[1], L.evec[2]);
    const Q4 zrot = mkq(L.zrot[0], L.zrot[1], L.zrot[2], L.zrot[3]);
    const V3 axis = mk3(L.axis[0], L.axis[1], L.axis[2]);
    Q4 cached;
    if (jtype == kJSpherical) cached = qmul(mkq(jp.x, jp.y, jp.z, -jp.w), zrot);
    else if (jtype == kJRevolute) { float s, c; sincosf(-0.5f * jp.x, &s, &c); cached = qmul(mkq(axis.x * s, axis.y * s, axis.z * s, c), zrot); }
    else cached = zrot;
    const M3 R = qmat(cached);
    const V3 r = dvec + mul(R, evec);
    const M3 Rwb = qmat(baseQuat);
    M3 Rwl = mul(R, Rwb);
    V3 pos = basePos + mulT(Rwl, r);
    for (int lv = 1; lv <= M.maxlevel; ++lv) {
        M3 pR; for (int k = 0; k < 9; ++k) pR.m[k] = T::shfl(Rwl.m[k], plane);
        V3 pp = T::shfl3(pos, plane);
        if (level == lv) { Rwl = mul(R, pR); pos = pp + mulT(Rwl, r); }
    }
    float ext_y;
    if (L.shape == kSSphere) ext_y = L.he[0];
    else {
        // world y extent = |row y of link->world basis| . half extents ; link->world basis row y = column y of Rwl
        float hx = L.shape == kSCapsule ? L.he[0] : L.he[0], hy = L.shape == kSCapsule ? L.he[0] + L.he[1] : L.he[1], hz = L.shape == kSCapsule ? L.he[0] : L.he[2];
        ext_y = fabsf(Rwl.m[1]) * hx + fabsf(Rwl.m[4]) * hy + fabsf(Rwl.m[7]) * hz;
    }
    float min_h = act ? (pos.y - ext_y) / M.scale - 0.001f : 1e30f;
    min_h = T::minf(min_h);
    const float min_violation = fminf(min_h, 0.f);
    if (min_violation < 0.f) basePos.y += -min_violation * M.scale;
    if constexpr (TASKV) {
        if (recovery) {   // all of the tile's shuffles are behind us: only lane 0 writes, the simulated state is left alone
            if (lane == 0) {
                tm[kTTimer] = 0.0; tm[kTTimerMax] = mt; tm[kTCtrl] = 0.0; tm[kTInitOff] = 0.0; tm[kTPrevAct] = 0.0;
                fl[kFNeedAction] = 1; fl[kFDone] = 0; fl[kFTerminate] = 0; fl[kFValid] = 1; fl[kFFallen] = 0; fl[kFUpdates] = 0; fl[7] = fl[7] + 1;
                st.taskx[static_cast<size_t>(env) * kTaskExtDoubles + kXRecover] = 1.0;
            }
            return;
        }
    }
    if (!doit) return;
    // ---- commit
    if (lane == 0) {
        reinterpret_cast<float4*>(sim)[0] = make_float4(basePos.x, basePos.y, basePos.z, 0.f);
        reinterpret_cast<float4*>(sim)[1] = make_float4(baseQuat.x, baseQuat.y, baseQuat.z, baseQuat.w);
        reinterpret_cast<float4*>(sim)[2] = make_float4(baseOmega.x, baseOmega.y, baseOmega.z, 0.f);
        reinterpret_cast<float4*>(sim)[3] = make_float4(baseVel.x, baseVel.y, baseVel.z, 0.f);
        // kinematic origin so that the clip's root coincides with the simulated root (SyncKinCharRoot)
        V3 rrp = qrot(orot, rp);
        tm[kTKin] = kt; tm[kTCtrl] = kt; tm[kTInitOff] = -kt; tm[kTPrevAct] = kt; tm[kTTimer] = 0.0; tm[kTTimerMax] = mt;
        tm[kTOrigin] = static_cast<double>(basePos.x / M.scale) - rrp.x; tm[kTOrigin + 1] = static_cast<double>(basePos.y / M.scale) - rrp.y;
        tm[kTOrigin + 2] = static_cast<double>(basePos.z / M.scale) - rrp.z;
        tm[kTOriginRot] = cth; tm[kTOriginRot + 1] = 0.0; tm[kTOriginRot + 2] = sth; tm[kTOriginRot + 3] = 0.0;
        fl[kFNeedAction] = 1; fl[kFDone] = 0; fl[kFTerminate] = 0; fl[kFValid] = 1; fl[kFFallen] = 0; fl[kFUpdates] = 0; fl[7] = fl[7] + 1;
        if constexpr (TASKV) st.clip[env] = new_clip;
    }
    if (!TASKV && act && st.hist) {
        // cSceneImitateAMP::InitHist (SceneImitateAMP.cpp:153-165): the kinematic character one query period before the controller time,
        // with the final origin (cKinCharacter::CalcPose / CalcVel, KinCharacter.cpp:363-406)
        const double tprev = kt - M.query_dt;
        DmJoint d = clip_joint(KM, L, frame_times, frames, frame_vel, tprev, lane == 0);
        if (lane == 0) {
            int idx, cyc; double bld;
            frame_index(KM, frame_times, tprev, idx, bld, cyc);
            if (KM.loop_motion) { d.p.x += cyc * KM.cycle_delta[0]; d.p.z += cyc * KM.cycle_delta[2]; }
            const V3 org = mk3(basePos.x / M.scale, basePos.y / M.scale, basePos.z / M.scale) - qrot(orot, rp);
            d.p = qrot(orot, d.p) + org;
            d.q = qmul(orot, d.q); if (d.q.w < 0) d.q = mkq(-d.q.x, -d.q.y, -d.q.z, -d.q.w);
            d.v = qrot(orot, d.v); d.w = qrot(orot, d.w);
        }
        hist_store(st.hist + static_cast<size_t>(env) * 2 * M.pose_dim, M.pose_dim, L, lane == 0, d);
    }
    if (act) {
        reinterpret_cast<float4*>(sim + 16)[lane] = jp;
        reinterpret_cast<float4*>(sim + 16 + 4 * nl)[lane] = jv;
        float4* mo = reinterpret_cast<float4*>(st.manifold + (static_cast<size_t>(env) * nl + lane) * kManifoldFloats);
        for (int k = 0; k < kManifoldFloats / 4; ++k) mo[k] = make_float4(0, 0, 0, 0);
    }
}

// ---------------------------------------------------------------------------------------------------------------- AMP task scenes
// One thread per environment; the per-update part of the task logic runs inside dm_step_kernel<.., TASK = true> (dm_task.cuh, dm_task_ext.cuh).

// After dm_reset_kernel: environments whose reset counter moved get cSceneTargetAMP::Reset's part (SceneTargetAMP.cpp:129-134):
// target timer, target position around the new root, heading 0 and a fresh speed (heading scene), previous-action COM 0.
__global__ void dm_task_reset_kernel(const DevModel* __restrict__ gm, DevState st, int num_envs) {
    const int env = blockIdx.x * blockDim.x + threadIdx.x;
    if (env >= num_envs) return;
    const DevModel& M = *gm;
    double* tk = st.task + static_cast<size_t>(env) * kTaskDoubles;
    double* tx = st.taskx + static_cast<size_t>(env) * kTaskExtDoubles;
    const int* fl = st.flags + static_cast<size_t>(env) * kFlagInts;
    if (static_cast<double>(fl[7]) == tk[kKResetSeen]) return;
    const float* sim = st.sim + static_cast<size_t>(env) * sim_stride(M.nl);
    const double* tm = st.time + static_cast<size_t>(env) * kTimeDoubles;
    const int kind = M.task_kind;
    TaskRng rng{M.task_seed, M.env_id_base + static_cast<unsigned long long>(env), tk + kKCounter};
    const double rx = static_cast<double>(sim[0]) / M.scale, rz = static_cast<double>(sim[2]) / M.scale;
    if (kind == kTaskHeadingGetup && tx[kXRecover] != 0.0) {   // recovery episode: target, timers of the task and the fallen character stay
        getup_recovery_reset(tk, tx);
        tx[kXRecover] = 0.0;
    } else if (kind == kTaskStrike) {   // cSceneTargetAMP::Reset with cSceneStrikeAMP::ResetTarget (SceneStrikeAMP.cpp:300-383); scene time 0
        task_timer_reset(M.task, tk, rng);
        strike_reset_target(M.task, M.taskx, tk, tx, rng, rx, rz, 0.0, M.test_mode != 0);
        tk[kKSpeed] = M.task.tar_speed;
        tk[kKPrevCom] = tk[kKPrevCom + 1] = tk[kKPrevCom + 2] = 0.0;
    } else {
        task_reset(task_base_kind(kind), M.task, tk, rng, rx, rz);
        if (kind == kTaskHeadingGetup) getup_reset(M.taskx, tx, tm[kTKin], st.ctab->info[st.clip[env]].is_getup != 0);   // SyncGetupTimer (:179-199)
    }
    tk[kKCom] = tk[kKCom + 1] = tk[kKCom + 2] = 0.0;
    tk[kKResetSeen] = static_cast<double>(fl[7]);
}

// RecordGoal ([N x goal_size]: 3, or 4 with the get-up / hit phase) and CalcReward ([N]) of the task scenes from the committed base state and the
// task blocks (SceneTargetAMP.cpp:3-80,185-215; SceneHeadingAMP.cpp:3-48,136-151; SceneHeadingAMPGetup.cpp:4-38,125-133; SceneStrikeAMP.cpp:9-190,407-430).
__global__ void dm_task_observe_kernel(const DevModel* __restrict__ gm, DevState st, float* __restrict__ goal, float* __restrict__ reward, int num_real_envs) {
    const int env = blockIdx.x * blockDim.x + threadIdx.x;
    if (env >= num_real_envs) return;
    const DevModel& M = *gm;
    const double* tk = st.task + static_cast<size_t>(env) * kTaskDoubles;
    const double* tx = st.taskx + static_cast<size_t>(env) * kTaskExtDoubles;
    const double* tm = st.time + static_cast<size_t>(env) * kTimeDoubles;
    const int* fl = st.flags + static_cast<size_t>(env) * kFlagInts;
    const float* sim = st.sim + static_cast<size_t>(env) * sim_stride(M.nl);
    const int kind = M.task_kind;
    const double rx = static_cast<double>(sim[0]) / M.scale, ry = static_cast<double>(sim[1]) / M.scale, rz = static_cast<double>(sim[2]) / M.scale;
    if (goal != nullptr) {
        // heading of the root joint (cKinTree::CalcHeading): the root rotation is the inverse of the stored world->base quaternion
        const double qx = -static_cast<double>(sim[4]), qy = -static_cast<double>(sim[5]), qz = -static_cast<double>(sim[6]), qw = static_cast<double>(sim[7]);
        const double hx = 1.0 - 2.0 * (qy * qy + qz * qz), hz = 2.0 * (qx * qz - qw * qy);   // rotate (1, 0, 0)
        const double heading = atan2(-hz, hx);
        double g[4] = {0.0, 0.0, 0.0, 0.0};
        int gs = 3;
        if (kind == kTaskStrike) { strike_goal(M.taskx, tk, tx, rx, rz, heading, tm[kTTimer], g); gs = 4; }
        else {
            task_goal(task_base_kind(kind), tk, rx, rz, heading, g);
            if (kind == kTaskHeadingGetup) { g[3] = getup_phase(M.taskx, tx); gs = 4; }
        }
        float* o = goal + static_cast<size_t>(env) * gs;
        for (int k = 0; k < gs; ++k) o[k] = static_cast<float>(g[k]);
    }
    if (reward != nullptr) {
        const double step_dur = tm[kTCtrl] - tm[kTPrevAct];
        double r;
        if (kind == kTaskStrike) r = strike_reward(M.task, M.taskx, tk, tx, fl[kFFallen] != 0, rx, rz, step_dur, M.test_mode != 0, fl[kFTerminate], tm[kTTimerMax], tm[kTTimer]);
        else if (kind == kTaskHeadingGetup && getup_active(M.taskx, tx)) r = getup_reward(M.taskx, ry, tx[kXHeadY]);
        else r = task_reward(task_base_kind(kind), M.task, tk, fl[kFFallen] != 0, rx, rz, step_dur);
        reward[env] = static_cast<float>(r);
    }
}

const ObserveKernel kObserveKernels[2][2] = {{dm_observe_kernel<16, kPolicyBlock, false>, dm_observe_kernel<16, kPolicyBlock, true>},
                                             {dm_observe_kernel<32, kPolicyBlock, false>, dm_observe_kernel<32, kPolicyBlock, true>}};
const ObserveDynKernel kObserveDynKernels[2][2] = {{dm_observe_dyn_kernel<16, kPolicyBlock, false>, dm_observe_dyn_kernel<16, kPolicyBlock, true>},
                                                   {dm_observe_dyn_kernel<32, kPolicyBlock, false>, dm_observe_dyn_kernel<32, kPolicyBlock, true>}};
const ResetKernel kResetKernels[2][2] = {{dm_reset_kernel<16, kPolicyBlock, false>, dm_reset_kernel<16, kPolicyBlock, true>},
                                         {dm_reset_kernel<32, kPolicyBlock, false>, dm_reset_kernel<32, kPolicyBlock, true>}};
const AmpObsKernel kAmpObsKernels[2][2] = {{dm_amp_obs_kernel<16, kPolicyBlock, false>, dm_amp_obs_kernel<16, kPolicyBlock, true>},
                                           {dm_amp_obs_kernel<32, kPolicyBlock, false>, dm_amp_obs_kernel<32, kPolicyBlock, true>}};
const AmpExpertKernel kAmpExpertKernels[2][2] = {{dm_amp_expert_sample_kernel<16, kPolicyBlock, false>, dm_amp_expert_sample_kernel<16, kPolicyBlock, true>},
                                                 {dm_amp_expert_sample_kernel<32, kPolicyBlock, false>, dm_amp_expert_sample_kernel<32, kPolicyBlock, true>}};

}  // namespace dmk
