// ORACLE -- TEST INFRASTRUCTURE ONLY.  Not shipped, not measured as the product.
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
// load this library.  The product path (deepmimic_b200/csrc) never calls into it.
//
// CPU restatement of DeepMimic's per-step simulation hot path for ONE environment, following the
// reference's order of operations file by file (each function cites the reference lines it follows):
//   cSceneImitate / cRLSceneSimChar / cSceneSimChar   R/DeepMimicCore/scenes/*.cpp
//   cSimCharacter / cSimBodyJoint / cSimBodyLink       R/DeepMimicCore/sim/*.cpp
//   cCtPDController / cImpPDController                 R/DeepMimicCore/sim/*.cpp
//   cKinCharacter / cMotion / cMotionController        R/DeepMimicCore/anim/*.cpp
//   cClipsController (clip datasets), cSceneImitateAMP, cSceneTargetAMP, cSceneHeadingAMP, cSceneHeadingAMPGetup, cSceneStrikeAMP (goal, task reward, target updates)
// DeepMimic's own math runs in double (rbd.hpp, omath.hpp); the Bullet 2.88 stage runs in float
// (bullet_mb.hpp).  PARITY UNPINNED: the reference ships no tests or golden vectors and Bullet is
// an un-vendored dependency, so this oracle is pinned only by the known-answer tests of
// SURVEY.md section 8(c) (tests/test_oracle_kat.py).
#include <array>
#include <cstdio>
#include <cstring>
#include <memory>
#include <string>

#include "bullet_mb.hpp"
#include "rbd.hpp"

namespace orc {

struct Oracle {
    dmh::SceneAssets sa;
    const CharModel* cm = nullptr;
    int nj = 0, ndof = 0;
    double scale = 1;
    // ---- cSimCharacter
    VecD pose, vel, pose0, vel0;
    std::vector<D3> link_lin_vel, link_ang_vel;  // cSimBodyLink::mLinVel / mAngVel (world frame, unscaled)
    std::vector<DQ> child_rot; std::vector<D3> child_pos;  // cSimBodyJoint::tParams::mChildRot / mChildPos
    DQ inv_root_attach_rot;
    BtMultiBody mb;
    std::vector<float> snap_frames;   // test tap: each link's collider worldBasis (row-major) and worldPos as of the last SetSnapshot
    BtContactSolverInfo info;
    double friction = 0.9 * 0.9;  // link 0.9 (SimCharacter.cpp:26) x ground 0.9 (Ground.cpp:17)
    // ---- cImpPDController
    RBDModel rbd;
    VecD kp, kd;
    std::vector<std::array<double, 4>> tar_theta;
    // ---- cCtController
    double ctrl_time = 0, init_time_offset = 0, prev_action_time = 0, cycle_period = 1;
    bool need_new_action = true;
    VecD action;
    std::vector<int> ctrl_off, ctrl_size;
    int action_size = 0;
    // ---- cKinCharacter + cMotionController / cClipsController (the active clip of the dataset; one clip with --kin_ctrl motion)
    int cur_clip = 0;
    std::vector<std::vector<double>> clip_frame_vel;
    std::vector<D3> clip_cycle_delta;
    const dmh::MotionClip& Mot() const { return sa.clips[cur_clip]; }
    const std::vector<double>& FrameVel() const { return clip_frame_vel[cur_clip]; }
    double kin_time = 0;
    D3 origin; DQ origin_rot;
    VecD kin_pose, kin_vel;
    D3 cycle_root_delta;
    // ---- cScene timer
    double timer_time = 0, timer_max = 0;
    VecD prev_pose, prev_vel;   // cSceneImitateAMP::mPrevPose / mPrevVel: sim pose / vel at the last applied action
    int mode = 0;  // 0 train, 1 test
    VecD joint_weights;
    // ---- AMP task scenes: cSceneTargetAMP / cSceneHeadingAMP (scenes/SceneTargetAMP.cpp, SceneHeadingAMP.cpp)
    enum SceneKind { kImitate = 0, kImitateAMP = 1, kTargetAMP = 2, kHeadingAMP = 3, kHeadingGetup = 4, kStrikeAMP = 5 };
    int scene_kind = kImitate;
    bool IsTask() const { return scene_kind == kTargetAMP || scene_kind == kHeadingAMP || scene_kind == kHeadingGetup || scene_kind == kStrikeAMP; }
    // cSceneStrikeAMP (scenes/SceneStrikeAMP.cpp): mTargetHit, mTargetHitTime; the target is a point in space (hits are detected by distance
    // and speed of the strike bodies, SceneStrikeAMP.cpp:440-481), so no prop bodies are involved
    bool target_hit = false;
    double target_hit_time = -1.0;
    bool IsHeading() const { return scene_kind == kHeadingAMP || scene_kind == kHeadingGetup; }
    // cSceneHeadingAMPGetup (scenes/SceneHeadingAMPGetup.cpp): mGetupTimer (max = mGetupTime), mGetupMotionFlags
    double getup_time = 0, getup_timer_time = 0;
    std::vector<char> getup_flags;
    bool CheckGettingUp() const { return !(getup_timer_time >= getup_time); }   // :296-299
    double tgt_timer_time = 0, tgt_timer_max = 0;   // mTargetTimer
    D3 target_pos;                                   // mTargetPos
    double target_speed = 1, target_heading = 0;     // mTargetSpeed, mTargetHeading
    D3 prev_action_com;                              // cDeepMimicCharController::mPrevActionCOM
    // The in-episode random draws of the task scenes come from a stateless counter-based stream shared with the CUDA path
    // (same splitmix64 finaliser as dm_policy.cu's u01): draw k of environment `task_env` is U01(task_seed, task_env, k).
    // The reference's std::mt19937 streams cannot be reproduced, so parity is defined on this stream.
    uint64_t task_seed = 0, task_env = 0, task_counter = 0;

    // =================================================================== construction
    void Init(const dmh::SceneAssets& assets) {
        sa = assets; cm = &sa.character; nj = cm->num_joints(); ndof = cm->pose_dim; scale = sa.cfg.world_scale;
        if (sa.cfg.scene == "imitate") scene_kind = kImitate;
        else if (sa.cfg.scene == "imitate_amp") scene_kind = kImitateAMP;
        else if (sa.cfg.scene == "target_amp") scene_kind = kTargetAMP;
        else if (sa.cfg.scene == "heading_amp") scene_kind = kHeadingAMP;
        else if (sa.cfg.scene == "heading_amp_getup") scene_kind = kHeadingGetup;
        else if (sa.cfg.scene == "strike_amp") scene_kind = kStrikeAMP;
        else throw std::runtime_error("oracle: scene '" + sa.cfg.scene + "' is not restated (imitate, imitate_amp, target_amp, heading_amp, heading_amp_getup, strike_amp)");
        if (scene_kind == kHeadingGetup) {   // Init: RecordGetupMotionFlags + CalcGetupTime (:87-98,221-243,262-287)
            getup_flags.assign(sa.clips.size(), 0);
            for (int id : sa.cfg.getup_motion_ids) {
                if (id < 0 || id >= static_cast<int>(sa.clips.size())) throw std::runtime_error("oracle: getup_motion_ids out of range");
                getup_flags[id] = 1; getup_time = std::max(getup_time, sa.clips[id].duration());
            }
            getup_timer_time = getup_time;   // ResetGetupTimer -> EndGetup
        }
        target_speed = sa.cfg.tar_speed;
        BuildKinMotion();
        BuildSimCharacter();
        BuildController();
        // cSceneImitate::CalcJointWeights (SceneImitate.cpp:236-248)
        joint_weights.assign(nj, 0.0);
        double sum = 0;
        for (int j = 0; j < nj; ++j) { joint_weights[j] = cm->joints[j].diff_weight; sum += std::fabs(joint_weights[j]); }
        for (auto& w : joint_weights) w /= sum;
        timer_max = sa.cfg.time_lim_max;
        prev_pose = pose0; prev_vel = vel0;
        Reset(0.0, 0.0, timer_max);
    }

    // cMotion::BuildFrameVel with cKinCharacter::CalcFrameVel (Motion.cpp:170-191, KinCharacter.cpp:433-437), for every clip of the dataset
    void BuildKinMotion() {
        clip_frame_vel.assign(sa.clips.size(), {});
        clip_cycle_delta.assign(sa.clips.size(), D3());
        for (size_t c = 0; c < sa.clips.size(); ++c) {
            const auto& mc = sa.clips[c];
            std::vector<double>& frame_vel = clip_frame_vel[c];
            frame_vel.assign(static_cast<size_t>(mc.num_frames) * ndof, 0.0);
            VecD f0(ndof), f1(ndof), v;
            for (int f = 0; f < mc.num_frames - 1; ++f) {
                double dt = mc.frame_times[f + 1] - mc.frame_times[f];
                std::copy(mc.frame(f), mc.frame(f) + ndof, f0.begin());
                std::copy(mc.frame(f + 1), mc.frame(f + 1) + ndof, f1.begin());
                CalcVel(*cm, f0, f1, dt, v);
                std::copy(v.begin(), v.end(), frame_vel.begin() + static_cast<size_t>(f) * ndof);
            }
            if (mc.num_frames > 1) std::copy(frame_vel.begin() + static_cast<size_t>(mc.num_frames - 2) * ndof, frame_vel.begin() + static_cast<size_t>(mc.num_frames - 1) * ndof,
                                             frame_vel.begin() + static_cast<size_t>(mc.num_frames - 1) * ndof);
            // cKinController::CalcCycleRootDelta (KinController.cpp:149-161)
            const double* fb = mc.frame(0); const double* fe = mc.frame(mc.num_frames - 1);
            clip_cycle_delta[c] = D3(fe[0] - fb[0], 0, fe[2] - fb[2]);
        }
        ActivateMotion(0);
        // cSceneImitate::BuildController (SceneImitate.cpp:250-264): the duration of the clip active at build time (a random one with
        // --kin_ctrl clips; only the phase input reads it, which the clip-dataset controllers do not enable)
        cycle_period = Mot().duration();
    }
    void ActivateMotion(int id) { cur_clip = id; cycle_root_delta = clip_cycle_delta[id]; }   // cClipsController::ActivateMotion (ClipsController.cpp:238-242)

    // cSimCharacter::BuildMultiBody / BuildConstraints / BuildJoints (SimCharacter.cpp:789-973,1036-1086)
    void BuildSimCharacter() {
        mb = BtMultiBody();
        mb.links.resize(nj);
        // CONVEX_DISTANCE_MARGIN; DMO_CAPSULE_MARGIN=0 reproduces round 1's margin-free capsule inertia for A/B runs of the behavioural pins
        const float capsule_inertia_margin = std::getenv("DMO_CAPSULE_MARGIN") ? static_cast<float>(std::atof(std::getenv("DMO_CAPSULE_MARGIN"))) : 0.04f;
        float fs = static_cast<float>(scale);
        mb.gravity = F3(static_cast<float>(sa.cfg.gravity.x * scale), static_cast<float>(sa.cfg.gravity.y * scale), static_cast<float>(sa.cfg.gravity.z * scale));  // cWorld::SetGravity (World.cpp:229-235)
        child_rot.resize(nj); child_pos.resize(nj);
        auto e2q = [](const dmh::V3& e) { return EulerToQuaternion(D3(e.x, e.y, e.z)); };
        auto toD3 = [](const dmh::V3& v) { return D3(v.x, v.y, v.z); };
        for (int j = 0; j < nj; ++j) {
            const auto& jd = cm->joints[j]; const auto& bd = cm->bodies[j];
            BtLink& L = mb.links[j];
            // collision shape at scaled size (World.cpp:335-377) and its local inertia
            float mass = static_cast<float>(bd.mass);
            L.mass = mass;
            if (bd.shape == dmh::kShapeBox) {
                L.shape = kBtBox;
                F3 he(fs * static_cast<float>(bd.param[0] * 0.5), fs * static_cast<float>(bd.param[1] * 0.5), fs * static_cast<float>(bd.param[2] * 0.5));
                L.halfExtents = he;  // getHalfExtentsWithMargin
                float lx = 2 * he.x, ly = 2 * he.y, lz = 2 * he.z;  // btBoxShape::calculateLocalInertia
                L.inertia = F3(mass / 12.0f * (ly * ly + lz * lz), mass / 12.0f * (lx * lx + lz * lz), mass / 12.0f * (lx * lx + ly * ly));
                L.manifold.breakingThreshold = 0.02f * length(he);
            } else if (bd.shape == dmh::kShapeCapsule) {
                L.shape = kBtCapsule;
                float r = static_cast<float>(scale * 0.5 * bd.param[0]);
                float hh = 0.5f * static_cast<float>(scale * bd.param[1]);  // btCapsuleShape(radius, height): halfHeight = 0.5*height
                L.halfExtents = F3(r, hh, 0);
                F3 he(r, r + hh, r);  // btCapsuleShape::calculateLocalInertia: bounding box of the capsule ...
                const float margin = capsule_inertia_margin;   // ... with CONVEX_DISTANCE_MARGIN (0.04) added to every half extent (Bullet 2.88)
                float lx = 2 * (he.x + margin), ly = 2 * (he.y + margin), lz = 2 * (he.z + margin);
                float sm = mass * 0.08333333f;
                L.inertia = F3(sm * (ly * ly + lz * lz), sm * (lx * lx + lz * lz), sm * (lx * lx + ly * ly));
                L.manifold.breakingThreshold = 0.02f * length(he);
            } else if (bd.shape == dmh::kShapeSphere) {
                L.shape = kBtSphere;
                float r = static_cast<float>(scale * 0.5 * bd.param[0]);
                L.halfExtents = F3(r, 0, 0);
                float e = 0.4f * mass * r * r;  // btSphereShape::calculateLocalInertia
                L.inertia = F3(e, e, e);
                L.manifold.breakingThreshold = 0.02f * length(F3(r, r, r));
            } else {
                assert(false && "oracle: unsupported body shape");
            }
            // frames ("arg so many transforms...", SimCharacter.cpp:819-845)
            DQ this_to_parent = e2q(jd.attach_theta);
            DQ body_to_this = e2q(bd.attach_theta);
            DQ this_to_body = qconj(body_to_this);
            DQ parent_body_to_parent; D3 parent_body_attach_pt;
            if (jd.parent >= 0) { parent_body_to_parent = e2q(cm->bodies[jd.parent].attach_theta); parent_body_attach_pt = toD3(cm->bodies[jd.parent].attach_pt); }
            DQ parent_to_parent_body = qconj(parent_body_to_parent);
            DQ body_to_parent_body = parent_to_parent_body * this_to_parent * body_to_this;
            DQ parent_body_to_body = qconj(body_to_parent_body);
            parent_body_attach_pt = QuatRotVec(parent_to_parent_body, parent_body_attach_pt);
            D3 joint_attach_pt = QuatRotVec(parent_to_parent_body, toD3(jd.attach_pt)) - parent_body_attach_pt;
            D3 body_attach_pt = QuatRotVec(qconj(body_to_this), toD3(bd.attach_pt));
            L.parent = jd.parent;
            L.zeroRotParentToThis = FQ(static_cast<float>(parent_body_to_body.x), static_cast<float>(parent_body_to_body.y), static_cast<float>(parent_body_to_body.z), static_cast<float>(parent_body_to_body.w));
            L.eVector = fs * F3(static_cast<float>(joint_attach_pt.x), static_cast<float>(joint_attach_pt.y), static_cast<float>(joint_attach_pt.z));
            L.dVector = fs * F3(static_cast<float>(body_attach_pt.x), static_cast<float>(body_attach_pt.y), static_cast<float>(body_attach_pt.z));
            bool is_root = jd.parent < 0;
            int jt = is_root ? dmh::kFixed : jd.type;  // floating base: root link is fixed to the massless base (SimCharacter.cpp:847-855)
            if (is_root && jd.type != dmh::kNone) assert(false && "oracle: only floating-base characters are restated");
            if (jt == dmh::kRevolute) {
                D3 axis = QuatRotVec(this_to_body, D3(0, 0, 1));
                L.jointType = kBtRevolute; L.dofCount = 1; L.posVarCount = 1;
                L.axisTop[0] = F3(static_cast<float>(axis.x), static_cast<float>(axis.y), static_cast<float>(axis.z));
                L.axisBottom[0] = cross(L.axisTop[0], L.dVector);
                L.jointPos[0] = 0;
                // cSimCharacter::BuildConstraints: note the reference compares lim_low[0] <= lim_high[1] (SimCharacter.cpp:958)
                if (jd.lim_low[0] <= jd.lim_high[1]) { L.hasLimit = true; L.limLow = static_cast<float>(jd.lim_low[0]); L.limHigh = static_cast<float>(jd.lim_high[0]); }
            } else if (jt == dmh::kSpherical) {
                L.jointType = kBtSpherical; L.dofCount = 3; L.posVarCount = 4;
                L.axisTop[0] = F3(1, 0, 0); L.axisTop[1] = F3(0, 1, 0); L.axisTop[2] = F3(0, 0, 1);
                for (int d = 0; d < 3; ++d) L.axisBottom[d] = cross(L.axisTop[d], L.dVector);
            } else if (jt == dmh::kFixed) {
                L.jointType = kBtFixed; L.dofCount = 0; L.posVarCount = 0;
            } else {
                assert(false && "oracle: unsupported joint type");
            }
            // cSimCharacter::BuildJoints: joint_to_child (SimCharacter.cpp:1052-1058)
            DT child_to_joint; child_to_joint.R = RotateMatEuler(toD3(bd.attach_theta)); child_to_joint.t = toD3(bd.attach_pt);
            DT joint_to_child = inv_rigid(child_to_joint);
            child_rot[j] = RotMatToQuaternion(joint_to_child.R);
            child_pos[j] = joint_to_child.t;
        }
        mb.finalize();
        inv_root_attach_rot = qconj(EulerToQuaternion(D3(cm->joints[0].attach_theta.x, cm->joints[0].attach_theta.y, cm->joints[0].attach_theta.z)));
        link_lin_vel.assign(nj, D3()); link_ang_vel.assign(nj, D3());
        // cCharacter::InitDefaultState (Character.cpp:387-394; KinTree.cpp:1159-1196)
        pose0.assign(ndof, 0.0); vel0.assign(ndof, 0.0);
        pose0[3] = 1;
        for (int j = 1; j < nj; ++j) if (cm->joints[j].type == dmh::kSpherical) pose0[cm->joints[j].param_offset] = 1;
        SetPose(pose0); SetVel(vel0);
    }

    // cCtPDController / cImpPDController / cPDController init (CtPDController.cpp:33-57, ImpPDController.cpp:25-38,97-127, PDController.cpp:99-112)
    void BuildController() {
        rbd.Init(*cm, D3(sa.cfg.gravity.x, sa.cfg.gravity.y, sa.cfg.gravity.z));
        kp.assign(ndof, 0.0); kd.assign(ndof, 0.0);
        tar_theta.assign(nj, {0, 0, 0, 0});
        for (int j = 1; j < nj; ++j) {
            const auto& jd = cm->joints[j];
            for (int k = 0; k < jd.param_size; ++k) { kp[jd.param_offset + k] = sa.ctrl.pd[j].kp; kd[jd.param_offset + k] = sa.ctrl.pd[j].kd; }
            VecD t(jd.param_size);
            for (int k = 0; k < jd.param_size; ++k) t[k] = sa.ctrl.pd[j].target_theta[k];
            SetTargetTheta(j, t);
        }
        // cCtController::BuildCtrlParamOffset (CtController.cpp:183-195) with cCtCtrlUtil::GetParamDimPD
        ctrl_off.assign(nj, 0); ctrl_size.assign(nj, 0);
        int off = 0;
        for (int j = 0; j < nj; ++j) {
            int sz = 0;
            if (j != 0) sz = (cm->joints[j].type == dmh::kSpherical) ? 3 : cm->joints[j].param_size;
            ctrl_off[j] = off; ctrl_size[j] = sz; off += sz;
        }
        action_size = off;
        action.assign(action_size, 0.0);
    }
    // cPDController::SetTargetTheta + PostProcessTargetPose (PDController.cpp:167-178,425-443)
    void SetTargetTheta(int j, const VecD& theta) {
        const auto& jd = cm->joints[j];
        VecD t = theta;
        if (jd.type == dmh::kSpherical) {
            double sq = 0; for (double x : t) sq += x * x;
            if (sq == 0) t[0] = 1; else { double n = std::sqrt(sq); for (auto& x : t) x /= n; }
        }
        for (int k = 0; k < jd.param_size; ++k) tar_theta[j][k] = t[k];
    }

    // =================================================================== cSimCharacter state <-> Bullet
    // cSimCharacter::SetPose (SimCharacter.cpp:725-763) + cSimBodyJoint::SetPose (SimBodyJoint.cpp:447-490)
    void SetPose(const VecD& p) {
        pose = p;
        float fs = static_cast<float>(scale);
        D3 rp = GetRootPos(p); DQ rr = GetRootRot(p);
        mb.basePos = fs * F3(static_cast<float>(rp.x), static_cast<float>(rp.y), static_cast<float>(rp.z));
        mb.baseQuat = inverse(FQ(static_cast<float>(rr.x), static_cast<float>(rr.y), static_cast<float>(rr.z), static_cast<float>(rr.w)));
        for (int j = 1; j < nj; ++j) {
            const auto& jd = cm->joints[j];
            BtLink& L = mb.links[j];
            if (jd.type == dmh::kRevolute) L.jointPos[0] = static_cast<float>(p[jd.param_offset]);
            else if (jd.type == dmh::kSpherical) {
                DQ q = child_rot[j] * pose_quat(p, jd.param_offset) * qconj(child_rot[j]);
                L.jointPos[0] = static_cast<float>(q.x); L.jointPos[1] = static_cast<float>(q.y); L.jointPos[2] = static_cast<float>(q.z); L.jointPos[3] = static_cast<float>(q.w);
            }
            L.updateCache();
        }
        mb.links[0].updateCache();
        mb.updateCollisionObjectWorldTransforms();  // UpdateLinkPos
        UpdateLinkVel();
    }
    // cSimCharacter::SetVel (SimCharacter.cpp:230-306) + cSimBodyJoint::SetVel (SimBodyJoint.cpp:492-545)
    void SetVel(const VecD& v) {
        vel = v;
        float fs = static_cast<float>(scale);
        D3 rv = GetRootVel(v), rw = GetRootAngVel(v);
        F3 bv = fs * F3(static_cast<float>(rv.x), static_cast<float>(rv.y), static_cast<float>(rv.z));
        mb.realBuf[0] = static_cast<float>(rw.x); mb.realBuf[1] = static_cast<float>(rw.y); mb.realBuf[2] = static_cast<float>(rw.z);
        mb.realBuf[3] = bv.x; mb.realBuf[4] = bv.y; mb.realBuf[5] = bv.z;
        for (int j = 1; j < nj; ++j) {
            const auto& jd = cm->joints[j];
            float* qd = mb.jointVel(j);
            if (jd.type == dmh::kRevolute) qd[0] = static_cast<float>(v[jd.param_offset]);
            else if (jd.type == dmh::kSpherical) {
                D3 w = QuatRotVec(child_rot[j], D3(v[jd.param_offset], v[jd.param_offset + 1], v[jd.param_offset + 2]));
                qd[0] = static_cast<float>(w.x); qd[1] = static_cast<float>(w.y); qd[2] = static_cast<float>(w.z);
            }
        }
        UpdateLinkVel();
    }
    // cSimObj::GetWorldTransform / GetPos / GetRotation (SimObj.cpp:15-99)
    DT BodyWorldTrans(int b) const {
        DT t;
        for (int i = 0; i < 3; ++i) for (int k = 0; k < 3; ++k) t.R.m[i][k] = mb.links[b].worldBasis.m[i][k];
        t.t = D3(mb.links[b].worldPos.x, mb.links[b].worldPos.y, mb.links[b].worldPos.z) / scale;
        return t;
    }
    D3 BodyPos(int b) const { return D3(mb.links[b].worldPos.x, mb.links[b].worldPos.y, mb.links[b].worldPos.z) / scale; }
    DQ BodyRot(int b) const { FQ q = fm3_get_rotation(mb.links[b].worldBasis); return DQ(q.w, q.x, q.y, q.z); }
    // cSimBodyJoint::BuildWorldTrans (SimBodyJoint.cpp:92-106)
    DT JointWorldTransSim(int j) const { DT jc; jc.R = RotateMatQuat(child_rot[j]); jc.t = child_pos[j]; return BodyWorldTrans(j) * jc; }
    D3 SimRootPos() const { return JointWorldTransSim(0).t; }                                                // SimCharacter.cpp:124-130
    DQ SimRootRot() const { return inv_root_attach_rot * RotMatToQuaternion(JointWorldTransSim(0).R); }      // SimCharacter.cpp:138-145
    // cSimBodyLink::GetLinearVelocity(local_pos) (SimBodyLink.cpp:49-57)
    D3 BodyPointVel(int b, const D3& local_pos) const { return link_lin_vel[b] + cross(link_ang_vel[b], QuatRotVec(BodyRot(b), local_pos)); }

    // cSimCharacter::UpdateLinkVel (SimCharacter.cpp:1219-1256) + cMultiBody::compTreeLinkVelocities (MultiBody.cpp:21-48)
    void UpdateLinkVel() {
        std::vector<F3> omega(nj + 1), v(nj + 1);
        omega[0] = quatRotate(mb.baseQuat, F3(mb.realBuf[0], mb.realBuf[1], mb.realBuf[2]));
        v[0] = quatRotate(mb.baseQuat, F3(mb.realBuf[3], mb.realBuf[4], mb.realBuf[5]));
        for (int i = 0; i < nj; ++i) {
            const BtLink& L = mb.links[i];
            FM3 R = fm3_from_quat(L.cachedRotParentToThis);
            omega[i + 1] = R * omega[L.parent + 1];
            v[i + 1] = -cross(L.cachedRVector, omega[i + 1]) + R * v[L.parent + 1];
            const float* qd = mb.jointVel(i);
            for (int d = 0; d < L.dofCount; ++d) { omega[i + 1] += qd[d] * L.axisTop[d]; v[i + 1] += qd[d] * L.axisBottom[d]; }
        }
        for (int b = 0; b < nj; ++b) {
            D3 cv = D3(v[b + 1].x, v[b + 1].y, v[b + 1].z) / scale;
            D3 co(omega[b + 1].x, omega[b + 1].y, omega[b + 1].z);
            DQ wr = BodyRot(b);
            link_lin_vel[b] = QuatRotVec(wr, cv);
            link_ang_vel[b] = QuatRotVec(wr, co);
        }
    }
    // cSimCharacter::BuildPose / BuildVel (SimCharacter.cpp:1428-1507) + cSimBodyJoint::BuildPose/BuildVel (SimBodyJoint.cpp:342-445)
    void BuildPoseVel() {
        D3 rp = SimRootPos(); DQ rr = SimRootRot();
        pose[0] = rp.x; pose[1] = rp.y; pose[2] = rp.z; pose[3] = rr.w; pose[4] = rr.x; pose[5] = rr.y; pose[6] = rr.z;
        // root vel = joint.CalcWorldVel() = child->GetLinearVelocity(child_pos); ang vel = child ang vel (SimBodyJoint.cpp:190-228)
        D3 rv = BodyPointVel(0, child_pos[0]), rw = link_ang_vel[0];
        vel[0] = rv.x; vel[1] = rv.y; vel[2] = rv.z; vel[3] = rw.x; vel[4] = rw.y; vel[5] = rw.z; vel[6] = 0;
        for (int j = 1; j < nj; ++j) {
            const auto& jd = cm->joints[j];
            const BtLink& L = mb.links[j];
            const float* qd = mb.jointVel(j);
            if (jd.type == dmh::kRevolute) { pose[jd.param_offset] = NormalizeAngle(L.jointPos[0]); vel[jd.param_offset] = qd[0]; }
            else if (jd.type == dmh::kSpherical) {
                DQ q(L.jointPos[3], L.jointPos[0], L.jointPos[1], L.jointPos[2]);
                q = qconj(child_rot[j]) * q * child_rot[j];
                if (q.w < 0) q = DQ(-q.w, -q.x, -q.y, -q.z);
                pose[jd.param_offset] = q.w; pose[jd.param_offset + 1] = q.x; pose[jd.param_offset + 2] = q.y; pose[jd.param_offset + 3] = q.z;
                D3 w = QuatRotVec(qconj(child_rot[j]), D3(qd[0], qd[1], qd[2]));
                vel[jd.param_offset] = w.x; vel[jd.param_offset + 1] = w.y; vel[jd.param_offset + 2] = w.z; vel[jd.param_offset + 3] = 0;
            }
        }
    }

    // =================================================================== kinematic character
    // cMotion::CalcIndexBlend (Motion.cpp:486-515)
    static void CalcIndexBlendOf(const dmh::MotionClip& mc, double time, int& idx, double& blend) {
        double max_time = mc.duration();
        if (!mc.loop) {
            if (time <= 0) { idx = 0; blend = 0; return; }
            if (time >= max_time) { idx = mc.num_frames - 2; blend = 1; return; }
        }
        int cycle = CalcCycleCountOf(mc, time);
        time -= cycle * max_time;
        auto it = std::upper_bound(mc.frame_times.begin(), mc.frame_times.end(), time);
        idx = static_cast<int>(it - mc.frame_times.begin()) - 1;
        double t0 = mc.frame_times[idx], t1 = mc.frame_times[idx + 1];
        blend = (time - t0) / (t1 - t0);
    }
    static int CalcCycleCountOf(const dmh::MotionClip& mc, double time) {  // Motion.cpp:476-484
        int count = static_cast<int>(std::floor(time / mc.duration()));
        if (!mc.loop) count = std::min(std::max(count, 0), 1);
        return count;
    }
    void CalcIndexBlend(double time, int& idx, double& blend) const { CalcIndexBlendOf(Mot(), time, idx, blend); }
    int CalcCycleCount(double time) const { return CalcCycleCountOf(Mot(), time); }
    double KinPhase(double t) const {  // cMotion::CalcPhase (Motion.cpp:27-40)
        double ph = t / Mot().duration();
        if (Mot().loop) ph -= std::floor(ph); else ph = std::min(std::max(ph, 0.0), 1.0);
        return ph;
    }
    // cKinCharacter::CalcPose (KinCharacter.cpp:363-386) <- cMotionController::CalcPose (MotionController.cpp:25-41) <- cMotion::CalcFrame
    void KinCalcPose(double time, VecD& out) const {
        int idx; double blend;
        CalcIndexBlend(time, idx, blend);
        blend = std::min(std::max(blend, 0.0), 1.0);  // cMathUtil::Saturate in cMotion::BlendFrames
        LerpPoses(*cm, Mot().frame(idx), Mot().frame(idx + 1), blend, out);
        if (Mot().loop) { D3 off = static_cast<double>(CalcCycleCount(time)) * cycle_root_delta; out[0] += off.x; out[1] += off.y; out[2] += off.z; }
        D3 rp = GetRootPos(out); DQ rr = GetRootRot(out);
        rr = StandardizeQuat(origin_rot * rr);
        rp = QuatRotVec(origin_rot, rp) + origin;
        out[0] = rp.x; out[1] = rp.y; out[2] = rp.z; out[3] = rr.w; out[4] = rr.x; out[5] = rr.y; out[6] = rr.z;
    }
    // cKinCharacter::CalcVel (KinCharacter.cpp:388-406) <- cMotion::CalcFrameVel (Motion.cpp:276-293)
    void KinCalcVel(double time, VecD& out) const {
        out.assign(ndof, 0.0);
        if (!(!Mot().loop && time >= Mot().duration())) {
            int idx; double blend;
            CalcIndexBlend(time, idx, blend);
            const double* v0 = &FrameVel()[static_cast<size_t>(idx) * ndof]; const double* v1 = &FrameVel()[static_cast<size_t>(idx + 1) * ndof];
            for (int k = 0; k < ndof; ++k) out[k] = (1.0 - blend) * v0[k] + blend * v1[k];
        }
        D3 rv = QuatRotVec(origin_rot, GetRootVel(out)), rw = QuatRotVec(origin_rot, GetRootAngVel(out));
        out[0] = rv.x; out[1] = rv.y; out[2] = rv.z; out[3] = rw.x; out[4] = rw.y; out[5] = rw.z;
    }
    void KinPose() { KinCalcPose(kin_time, kin_pose); KinCalcVel(kin_time, kin_vel); }  // cKinCharacter::Pose (KinCharacter.cpp:199-211)
    void KinMoveOrigin(const D3& delta) { origin += delta; kin_pose[0] += delta.x; kin_pose[1] += delta.y; kin_pose[2] += delta.z; }  // KinCharacter.cpp:260-271
    // cKinCharacter::RotateOrigin (KinCharacter.cpp:285-327)
    void KinRotateOrigin(const DQ& rot) {
        origin_rot = qnormalized(rot * origin_rot);
        D3 rp = GetRootPos(kin_pose);
        origin = rp + QuatRotVec(rot, origin - rp);
        DQ rr = qnormalized(rot * GetRootRot(kin_pose));
        kin_pose[3] = rr.w; kin_pose[4] = rr.x; kin_pose[5] = rr.y; kin_pose[6] = rr.z;
        D3 v = QuatRotVec(rot, GetRootVel(kin_vel)), w = QuatRotVec(rot, GetRootAngVel(kin_vel));
        kin_vel[0] = v.x; kin_vel[1] = v.y; kin_vel[2] = v.z; kin_vel[3] = w.x; kin_vel[4] = w.y; kin_vel[5] = w.z;
    }

    // =================================================================== reset (SURVEY 3d)
    // cSceneSimChar::ResetScene (SceneSimChar.cpp:628-644) with the RNG draws injected: kin_time ~ U(0,dur),
    // rand_theta ~ U(-pi,pi) (only if --enable_rand_rot_reset), max_time ~ U(time_lim_min, time_lim_max).
    // With --kin_ctrl clips the controller also draws a new clip (cClipsController::Reset, ClipsController.cpp:37-46): injected as
    // `clip` (< 0 keeps the active one).  Note the reference draws rand_kin_time from U(0, duration of the PREVIOUS clip) because
    // CalcRandKinResetTime runs before kin_char->Reset() (SceneImitate.cpp:331-338); a sampler that wants the reference's
    // distribution must do the same.
    void Reset(double rand_kin_time, double rand_theta, double max_time, int clip = -1) {
        if (scene_kind == kHeadingGetup && ActivateRecoveryEpisode()) { ResetRecoveryEpisode(max_time); return; }   // SceneHeadingAMPGetup.cpp:111-123
        if (clip >= 0) ActivateMotion(clip);
        timer_time = 0;
        timer_max = (mode == 1) ? sa.cfg.time_end_lim_max : max_time;  // cRLSceneSimChar::ResetTimers (RLSceneSimChar.cpp:277-284)
        mb.clearContacts();                                            // cWorld::Reset (World.cpp:75-91)
        for (auto& L : mb.links) { L.appliedForce = F3(); L.appliedTorque = F3(); L.jointTorque[0] = L.jointTorque[1] = L.jointTorque[2] = 0; }
        // cSceneImitate::ResetCharacters (SceneImitate.cpp:320-329)
        SetPose(pose0); SetVel(vel0);                                  // cCharacter::Reset
        ctrl_time = 0; need_new_action = true; prev_action_time = 0; init_time_offset = 0;  // cDeepMimicCharController::ResetParams / cCtController::ResetParams
        prev_action_com = D3();                                                             // DeepMimicCharController.cpp:227-228
        // ResetKinChar (SceneImitate.cpp:331-349)
        origin_rot = DQ(); origin = D3();
        kin_time = rand_kin_time;
        KinPose();
        if (sa.cfg.enable_rand_rot_reset) KinRotateOrigin(AxisAngleToQuaternion(D3(0, 1, 0), rand_theta));  // EulerToQuaternion((0,theta,0))
        // SyncCharacters (SceneImitate.cpp:351-368)
        SetPose(kin_pose); SetVel(kin_vel);
        ctrl_time = kin_time; prev_action_time = kin_time; init_time_offset = -kin_time;  // cCtController::SetInitTime (CtController.cpp:144-150)
        // InitCharacterPos -> SetCharRandPlacement -> SetRootTransform (SceneSimChar.cpp:478-531, SimCharacter.cpp:185-202): x,z := 0
        {
            VecD p = pose;
            p[0] = 0; p[2] = 0;  // rand_pos = (0, ground_h = 0, 0), height and rotation kept (delta_rot = identity)
            SetPose(p); SetVel(vel);
        }
        ResolveCharGroundIntersect();
        // SyncKinCharRoot (SceneImitate.cpp:386-418)
        {
            if (sa.cfg.sync_char_root_rot) {
                // cCharacter::RotateRoot -> virtual SetRootRotation -> cKinCharacter::SetRootRotation -> RotateOrigin (Character.cpp:210-216,
                // KinCharacter.cpp:243-248,285-327): the heading difference goes into the kinematic character's ORIGIN rotation and persists
                double sim_heading = CalcHeading(SimRootRot()), kin_heading = CalcHeading(GetRootRot(kin_pose));
                KinRotateOrigin(AxisAngleToQuaternion(D3(0, 1, 0), sim_heading - kin_heading));
            }
            KinMoveOrigin(SimRootPos() - GetRootPos(kin_pose));  // cKinCharacter::SetRootPos (KinCharacter.cpp:239-244)
        }
        // cSceneImitateAMP::Reset (SceneImitateAMP.cpp:58-68).  cSceneTargetAMP::Reset calls cSceneImitate::Reset directly
        // (SceneTargetAMP.cpp:129-134), so the task scenes keep the history of the last applied action across resets.
        if (!IsTask()) InitHist();
        if (IsTask()) { TargetTimerReset(); ResetTarget(); }   // SceneTargetAMP.cpp:132-133
        if (scene_kind == kHeadingGetup) {
            // ResetTimers (virtual, inside the base reset) -> ResetGetupTimer -> EndGetup; then SyncGetupTimer: an episode that starts in a
            // get-up clip starts getting up at the clip's time (SceneHeadingAMPGetup.cpp:161-165,179-199)
            getup_timer_time = getup_time;
            if (getup_flags[cur_clip]) getup_timer_time = kin_time;
        }
    }
    // cSceneHeadingAMPGetup::ActivateRecoveryEpisode (:301-317).  The member mIsRecoveryEpisode is shadowed by a local in Reset() and never
    // becomes true, so the "!mIsRecoveryEpisode" guard never blocks.
    bool ActivateRecoveryEpisode() {
        if (mode == 0 && sa.cfg.recover_episode_prob > 0.0 && CheckTerminate() == 1) return FlipCoin(sa.cfg.recover_episode_prob);
        return false;
    }
    // cSceneHeadingAMPGetup::ResetRecoveryEpisode (:40-58): the fallen character stays where it is; only the timers and the controller restart
    void ResetRecoveryEpisode(double max_time) {
        timer_time = 0; timer_max = (mode == 1) ? sa.cfg.time_end_lim_max : max_time;   // ResetTimers
        getup_timer_time = 0;                                                            // ResetGetupTimer (-> EndGetup) then BeginGetup
        ctrl_time = 0; need_new_action = true; prev_action_time = 0; init_time_offset = 0; prev_action_com = D3();   // ctrl->Reset()
    }
    // cSceneSimChar::ResolveCharGroundIntersect (SceneSimChar.cpp:542-583); AABBs from btCollisionShape::getAabb [B288-mem]
    void ResolveCharGroundIntersect() {
        const double pad = 0.001;
        double min_violation = 0;
        for (int b = 0; b < nj; ++b) {
            const BtLink& L = mb.links[b];
            FM3 ab = fm3_absolute(L.worldBasis);
            F3 he;
            if (L.shape == kBtSphere) he = F3(L.halfExtents.x, L.halfExtents.x, L.halfExtents.x);
            else if (L.shape == kBtCapsule) he = F3(L.halfExtents.x, L.halfExtents.x + L.halfExtents.y, L.halfExtents.x);
            else he = L.halfExtents;
            float ext_y = (L.shape == kBtSphere) ? L.halfExtents.x : (ab.m[1][0] * he.x + ab.m[1][1] * he.y + ab.m[1][2] * he.z);
            double min_h = (L.worldPos.y - ext_y) / scale;
            min_violation = std::min(min_violation, min_h - pad);
        }
        if (min_violation < 0) { VecD p = pose; p[1] += -min_violation; SetPose(p); }
    }

    // =================================================================== per-update hot loop (SURVEY 3b)
    // cSceneSimChar::Update (SceneSimChar.cpp:136-161)
    void Update(double dt) {
        timer_time += dt;                    // cScene::Update -> UpdateTimers
        if (scene_kind == kHeadingGetup) getup_timer_time += dt;   // cSceneHeadingAMPGetup::UpdateTimers (:167-171)
        if (dt < 0) return;
        UpdateKinChar(dt);                   // cSceneImitate::UpdateCharacters (SceneImitate.cpp:300-304)
        UpdateSimChar(dt);
        // cWorld::Update (World.cpp:93-104)
        float timestep = static_cast<float>(std::max(0.0, dt));
        float sub = timestep / sa.cfg.num_sim_substeps;
        mb.stepSimulation(timestep, sa.cfg.num_sim_substeps, sub, info, static_cast<float>(friction));
        // cSimCharacter::PostUpdate (SimCharacter.cpp:112-122)
        UpdateLinkVel();
        BuildPoseVel();
        need_new_action = CheckNextInterval(dt, ctrl_time + init_time_offset, 1.0 / sa.ctrl.query_rate);  // CtController.cpp:221-227
        if (IsTask()) {   // cSceneTargetAMP::Update (SceneTargetAMP.cpp:136-145)
            UpdateTarget(dt);
            if (tgt_timer_time >= tgt_timer_max) TargetTimerReset();
        }
        if (scene_kind == kHeadingGetup && mode == 1) {   // UpdateTestGetup (:245-254): a fall in test mode starts a get-up instead of ending the episode
            if (ContactFall() && !CheckGettingUp()) getup_timer_time = 0;
        }
    }
    // cSceneImitate::UpdateKinChar + SyncKinCharNewCycle (SceneImitate.cpp:306-318,420-444)
    void UpdateKinChar(double dt) {
        double prev_phase = KinPhase(kin_time);
        kin_time += dt;
        KinPose();
        double curr_phase = KinPhase(kin_time);
        if (curr_phase < prev_phase) {
            if (sa.cfg.sync_char_root_rot) {   // RotateRoot -> RotateOrigin, as in Reset's SyncKinCharRoot
                double sim_heading = CalcHeading(SimRootRot()), kin_heading = CalcHeading(GetRootRot(kin_pose));
                KinRotateOrigin(AxisAngleToQuaternion(D3(0, 1, 0), sim_heading - kin_heading));
            }
            if (sa.cfg.sync_char_root_pos) {
                D3 sim_root = SimRootPos(), kin_root = GetRootPos(kin_pose);
                kin_root.x = sim_root.x; kin_root.z = sim_root.z;
                double dh = kin_root.y - origin.y;
                kin_root.y = 0 + dh;
                KinMoveOrigin(kin_root - GetRootPos(kin_pose));
            }
        }
    }
    // cSimCharacter::Update -> cCtPDController -> cImpPDController::CalcControlForces -> joint.ApplyTau
    void UpdateSimChar(double dt) {
        ctrl_time += dt;  // cDeepMimicCharController::UpdateCalcTau (DeepMimicCharController.cpp:71-78)
        if (need_new_action) { prev_action_time = ctrl_time; prev_action_com = CalcCOM(); need_new_action = false; UpdateHist(); }  // HandleNewAction (DeepMimicCharController.cpp:262-267) -> cSceneImitateAMP::NewActionUpdate
        VecD tau(ndof, 0.0);
        if (dt > 0) {
            rbd.Update(pose, vel);                         // cImpPDController::UpdateRBDModel (ImpPDController.cpp:129-134)
            CalcControlForces(dt, tau);
        }
        // cSimCharacter::ApplyControlForces + UpdateJoints -> cSimBodyJoint::ApplyTau* (SimCharacter.cpp:698-715,1201-1212; SimBodyJoint.cpp:636-695)
        for (int j = 1; j < nj; ++j) {
            const auto& jd = cm->joints[j];
            BtLink& L = mb.links[j];
            double lim = jd.torque_lim;
            if (jd.type == dmh::kRevolute) {
                D3 t(0, 0, tau[jd.param_offset]);
                double mag = norm(t);
                if (mag > lim) t = t * (lim / mag);
                L.jointTorque[0] += static_cast<float>(scale * scale * t.z);
            } else if (jd.type == dmh::kSpherical) {
                D3 t(tau[jd.param_offset], tau[jd.param_offset + 1], tau[jd.param_offset + 2]);
                double mag = norm(t);
                if (mag > lim) t = t * (lim / mag);
                t = QuatRotVec(child_rot[j], t);
                L.jointTorque[0] += static_cast<float>(scale * scale * t.x);
                L.jointTorque[1] += static_cast<float>(scale * scale * t.y);
                L.jointTorque[2] += static_cast<float>(scale * scale * t.z);
            }
        }
    }
    // cImpPDController::CalcControlForces (ImpPDController.cpp:136-195) -- Stable PD
    void CalcControlForces(double t, VecD& out_tau) {
        VecD tar_pose(ndof, 0.0), tar_vel(ndof, 0.0);
        for (int j = 1; j < nj; ++j) for (int k = 0; k < cm->joints[j].param_size; ++k) tar_pose[cm->joints[j].param_offset + k] = tar_theta[j][k];
        std::vector<double> M = rbd.M;
        for (int i = 0; i < ndof; ++i) M[static_cast<size_t>(i) * ndof + i] += t * kd[i];
        VecD pose_inc;
        VelToPoseDiff(*cm, pose, vel, pose_inc);
        for (int i = 0; i < ndof; ++i) pose_inc[i] = pose[i] + t * pose_inc[i];
        PostProcessPose(*cm, pose_inc);
        VecD pose_err;
        CalcVel(*cm, pose_inc, tar_pose, 1, pose_err);
        VecD acc(ndof), vel_err(ndof);
        for (int i = 0; i < ndof; ++i) { vel_err[i] = tar_vel[i] - vel[i]; acc[i] = kp[i] * pose_err[i] + kd[i] * vel_err[i] - rbd.C[i]; }
        acc = SolveSymmetric(M, ndof, acc);
        for (int i = 0; i < ndof; ++i) out_tau[i] += kp[i] * pose_err[i] + kd[i] * (vel_err[i] - t * acc[i]);
    }

    // =================================================================== 30 Hz policy interface (SURVEY 3c)
    // cCtPDController::ApplyAction / SetPDTargets / ConvertActionToTargetPose (CtPDController.cpp:97-101,115-166)
    void SetAction(const double* a) {
        for (int i = 0; i < action_size; ++i) action[i] = a[i];
        for (int j = 1; j < nj; ++j) {
            const auto& jd = cm->joints[j];
            if (jd.type == dmh::kSpherical) {
                D3 em(a[ctrl_off[j]], a[ctrl_off[j] + 1], a[ctrl_off[j] + 2]);
                double len = norm(em), max_len = 2.0 * M_PI;
                if (len > max_len) em = em * (max_len / len);
                DQ q = ExpMapToQuaternion(em);
                SetTargetTheta(j, {q.w, q.x, q.y, q.z});
            } else if (ctrl_size[j] > 0) {
                VecD t(ctrl_size[j]);
                for (int k = 0; k < ctrl_size[j]; ++k) t[k] = a[ctrl_off[j] + k];
                SetTargetTheta(j, t);
            }
        }
    }
    int StateSize() const { return (sa.ctrl.enable_phase_input ? 1 : 0) + nj * 9 + 1 + nj * 6; }  // CtController.cpp:41-46,300-330
    // cCtController::RecordState / BuildStatePose / BuildStateVel / BuildStatePhase (CtController.cpp:281-293,373-478)
    // =================================================================== AMP observations (cSceneImitateAMP, SceneImitateAMP.cpp)
    void InitHist() {   // :153-165 -- the kinematic character one query period before the controller time
        const double t = ctrl_time - 1.0 / sa.ctrl.query_rate;
        KinCalcPose(t, prev_pose); KinCalcVel(t, prev_vel);
    }
    void UpdateHist() { prev_pose = pose; prev_vel = vel; }   // :167-172
    int AmpObsPoseSize() const {   // :214-242
        int size = 1 + 6 + 3 * static_cast<int>(EndEffectors().size());
        for (int j = 1; j < nj; ++j) size += (cm->joints[j].type == dmh::kSpherical) ? 6 : cm->joints[j].param_size;
        return size;
    }
    int AmpObsVelSize() const { return ndof - cm->joints[0].param_size + 3 + 3; }   // :244-258
    int AmpObsSize() const { return 2 * (AmpObsPoseSize() + AmpObsVelSize()); }    // :75-84
    std::vector<int> EndEffectors() const { std::vector<int> e; for (int j = 0; j < nj; ++j) if (cm->joints[j].is_end_eff) e.push_back(j); return e; }
    int RecordAMPObsPose(const VecD& p, double ground_h, const DQ& ref_rot, int off, double* out) const {   // :296-365
        int o = off;
        const D3 root_pos = GetRootPos(p);
        DQ root_rot = GetRootRot(p);
        out[o++] = root_pos.y - ground_h;
        if (sa.cfg.enable_amp_obs_local_root) root_rot = ref_rot * root_rot;
        D3 nrm = QuatRotVec(root_rot, D3(0, 1, 0)), tan = QuatRotVec(root_rot, D3(1, 0, 0));   // cMathUtil::CalcNormalTangent (MathUtil.cpp:617-623)
        out[o] = nrm.x; out[o + 1] = nrm.y; out[o + 2] = nrm.z; out[o + 3] = tan.x; out[o + 4] = tan.y; out[o + 5] = tan.z; o += 6;
        for (int j = 1; j < nj; ++j) {
            const auto& jd = cm->joints[j];
            if (jd.type == dmh::kSpherical) {
                DQ q(p[jd.param_offset], p[jd.param_offset + 1], p[jd.param_offset + 2], p[jd.param_offset + 3]);
                D3 n = QuatRotVec(q, D3(0, 1, 0)), t = QuatRotVec(q, D3(1, 0, 0));
                out[o] = n.x; out[o + 1] = n.y; out[o + 2] = n.z; out[o + 3] = t.x; out[o + 4] = t.y; out[o + 5] = t.z; o += 6;
            } else for (int k = 0; k < jd.param_size; ++k) out[o++] = p[jd.param_offset + k];
        }
        for (int e : EndEffectors()) {   // cKinTree::CalcBodyPartPos (KinTree.cpp:272-281): joint_to_world * BodyJointTrans.col(3)
            const DT jw = JointWorldTrans(*cm, p, e);
            D3 bp = jw.R * BodyJointTrans(*cm, e).t + jw.t;
            bp = QuatRotVec(ref_rot, bp - root_pos);
            out[o] = bp.x; out[o + 1] = bp.y; out[o + 2] = bp.z; o += 3;
        }
        return o - off;
    }
    int RecordAMPObsVel(const VecD& v, const DQ& ref_rot, int off, double* out) const {   // :367-397
        int o = off;
        D3 rv = GetRootVel(v), rw = GetRootAngVel(v);
        if (sa.cfg.enable_amp_obs_local_root) { rv = QuatRotVec(ref_rot, rv); rw = QuatRotVec(ref_rot, rw); }
        out[o] = rv.x; out[o + 1] = rv.y; out[o + 2] = rv.z; out[o + 3] = rw.x; out[o + 4] = rw.y; out[o + 5] = rw.z; o += 6;
        const int rs = cm->joints[0].param_size;
        for (int k = rs; k < ndof; ++k) out[o++] = v[k];
        return o - off;
    }
    void BuildAMPObs(const VecD& pp, const VecD& pv, const VecD& p, const VecD& v, double ground_h, double* out) const {   // :279-294
        const DQ ref_rot = AxisAngleToQuaternion(D3(0, 1, 0), -CalcHeading(GetRootRot(p)));   // cKinTree::CalcHeadingRot (KinTree.cpp:1629-1635)
        int o = 0;
        o += RecordAMPObsPose(p, ground_h, ref_rot, o, out);
        o += RecordAMPObsPose(pp, ground_h, ref_rot, o, out);
        o += RecordAMPObsVel(v, ref_rot, o, out);
        o += RecordAMPObsVel(pv, ref_rot, o, out);
    }
    void RecordAMPObsAgent(double* out) const { BuildAMPObs(prev_pose, prev_vel, pose, vel, 0.0, out); }   // :101-113 (flat ground at 0)
    // :115-140 with the random mocap time injected; cMotion::CalcFrame / CalcFrameVel of the raw clip (no origin, no cycle offset)
    void MotionCalcFrame(int clip, double time, VecD& p, VecD& v) const {
        const dmh::MotionClip& mc = sa.clips[clip];
        const std::vector<double>& fv = clip_frame_vel[clip];
        int idx; double blend;
        CalcIndexBlendOf(mc, time, idx, blend);
        const double b = std::min(std::max(blend, 0.0), 1.0);
        LerpPoses(*cm, mc.frame(idx), mc.frame(idx + 1), b, p);
        v.assign(ndof, 0.0);
        if (!(!mc.loop && time >= mc.duration())) {
            const double* v0 = &fv[static_cast<size_t>(idx) * ndof]; const double* v1 = &fv[static_cast<size_t>(idx + 1) * ndof];
            for (int k = 0; k < ndof; ++k) v[k] = (1.0 - blend) * v0[k] + blend * v1[k];
        }
    }
    // clip < 0: the active clip (cSceneImitateAMP::SampleExpertMotion without a clips controller, :260-277); otherwise the clip the
    // dataset sampler drew (cClipsController::SampleMotionID) with rand_kin_time ~ U(0, that clip's duration)
    void RecordAMPObsExpert(int clip, double rand_kin_time, double* out) const {
        VecD p, v, pp, pv;
        const int c = clip < 0 ? cur_clip : clip;
        MotionCalcFrame(c, rand_kin_time, p, v);
        MotionCalcFrame(c, rand_kin_time - 1.0 / sa.ctrl.query_rate, pp, pv);
        BuildAMPObs(pp, pv, p, v, origin.y, out);
    }

    void RecordState(double* out) const {
        int ph = sa.ctrl.enable_phase_input ? 1 : 0;
        // cKinTree::BuildOriginTrans (KinTree.cpp:1651-1664) on the sim character's pose
        D3 rpose = GetRootPos(pose);
        double heading = CalcHeading(GetRootRot(pose));
        DM3 Rh = RotateMatAxis(D3(0, 1, 0), -heading);
        D3 org(rpose.x, 0, rpose.z);
        auto origin_apply = [&](const D3& p) { return Rh * (p - org); };
        DQ origin_quat = RotMatToQuaternion(Rh);
        D3 root_pos = SimRootPos();
        double ground_h = 0;
        D3 root_pos_rel = root_pos; root_pos_rel.y -= ground_h;
        root_pos_rel = origin_apply(root_pos_rel);
        if (ph) { double p = std::fmod(ctrl_time / cycle_period, 1.0); out[0] = (p < 0) ? 1 + p : p; }  // cCtController::GetPhase (CtController.cpp:152-159)
        double* op = out + ph;
        op[0] = root_pos_rel.y;
        for (int i = 0; i < nj; ++i) {
            D3 cp = BodyPos(i); cp.y -= ground_h;
            if (!sa.ctrl.record_world_root_pos || i != 0) cp = origin_apply(cp) - root_pos_rel;
            DQ cq = BodyRot(i);
            if (!sa.ctrl.record_world_root_rot || i != 0) cq = origin_quat * cq;
            D3 nrm = QuatRotVec(cq, D3(0, 1, 0)), tan = QuatRotVec(cq, D3(1, 0, 0));  // cMathUtil::CalcNormalTangent (MathUtil.cpp:617-623)
            double* o = op + 1 + 9 * i;
            o[0] = cp.x; o[1] = cp.y; o[2] = cp.z; o[3] = nrm.x; o[4] = nrm.y; o[5] = nrm.z; o[6] = tan.x; o[7] = tan.y; o[8] = tan.z;
        }
        double* ov = op + 1 + 9 * nj;
        for (int i = 0; i < nj; ++i) {
            D3 v = link_lin_vel[i], w = link_ang_vel[i];
            if (!sa.ctrl.record_world_root_rot || i != 0) { v = Rh * v; w = Rh * w; }
            double* o = ov + 6 * i;
            o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = w.x; o[4] = w.y; o[5] = w.z;
        }
    }
    // cContactManager::Update + cSimCharacter::CheckFallContact (ContactManager.cpp:62-118; SimCharacter.cpp:1509-1525)
    bool BodyInContact(int b) const {
        float tol = static_cast<float>(0.001 * scale);
        const BtManifold& m = mb.links[b].manifold;
        for (int k = 0; k < m.n; ++k) if (m.pt[k].distance1 <= tol) return true;
        return false;
    }
    bool ContactFall() const {   // cSimCharacter::HasFallen: any fall-contact body touching the ground
        if (sa.cfg.enable_char_contact_fall) for (int b = 0; b < nj; ++b) if (cm->bodies[b].fall_contact && BodyInContact(b)) return true;
        return false;
    }
    bool HasFallen() const {  // cSceneImitate::HasFallen (SceneImitate.cpp:466-475) -> cSceneSimChar::HasFallen (SceneSimChar.cpp:822-841)
        // cSceneHeadingAMPGetup::HasFallenContact (:256-265): no contact fall while getting up
        bool fallen = (scene_kind == kHeadingGetup && CheckGettingUp()) ? false : ContactFall();
        if (sa.cfg.enable_root_rot_fail) fallen |= QuatDiffTheta(SimRootRot(), GetRootRot(kin_pose)) > 0.5 * M_PI;
        return fallen;
    }
    // cSceneImitate::CalcReward / CalcRewardImitate (SceneImitate.cpp:7-127,163-175)
    // force_imitate: cSceneImitate::CalcRewardImitate whatever the scene (the task scenes inherit it; BASELINE.json config 5 records it next to
    // the AMP observations) -- against the kinematic character, i.e. the active clip of the dataset
    double CalcReward(double* dbg = nullptr, bool force_imitate = false) const {
        if (!force_imitate && scene_kind == kTargetAMP) return CalcRewardTarget();
        if (!force_imitate && scene_kind == kStrikeAMP) return CalcRewardStrike();
        if (!force_imitate && scene_kind == kHeadingGetup && CheckGettingUp()) {   // cSceneHeadingAMPGetup::CalcRewardGetup (:18-38), flat ground at 0
            const double root_h = std::min(std::max(SimRootPos().y / sa.cfg.getup_height_root, 0.0), 1.0);
            const double head_h = std::min(std::max(BodyPos(sa.cfg.head_id).y / sa.cfg.getup_height_head, 0.0), 1.0);
            return 0.2 * root_h + 0.8 * head_h;
        }
        if (!force_imitate && IsHeading()) return CalcRewardHeading();
        if (HasFallen()) return 0;
        double pose_w = 0.5, vel_w = 0.05, end_eff_w = 0.15, root_w = 0.2, com_w = 0.1;
        double total_w = pose_w + vel_w + end_eff_w + root_w + com_w;
        pose_w /= total_w; vel_w /= total_w; end_eff_w /= total_w; root_w /= total_w; com_w /= total_w;
        const double pose_scale = 2.0 / 15 * nj, vel_scale = 0.1 / 15 * nj, end_eff_scale = 10, root_scale = 5, com_scale = 10, err_scale = 1;
        const VecD& pose0_ = pose; const VecD& vel0_ = vel; const VecD& pose1 = kin_pose; const VecD& vel1 = kin_vel;
        auto origin_trans_of = [](const VecD& p) {
            double heading = CalcHeading(GetRootRot(p));
            DM3 Rh = RotateMatAxis(D3(0, 1, 0), -heading);
            D3 org(p[0], 0, p[2]);
            return std::make_pair(Rh, org);
        };
        auto ot0 = origin_trans_of(pose0_), ot1 = origin_trans_of(pose1);
        // sim COM velocity: mass-weighted link velocities (SimCharacter.cpp:386-428)
        D3 com_vel0; double tm = 0;
        for (int b = 0; b < nj; ++b) { com_vel0 += cm->bodies[b].mass * link_lin_vel[b]; tm += cm->bodies[b].mass; }
        com_vel0 = com_vel0 / tm;
        D3 com1, com_vel1;
        CalcCoM(*cm, pose1, vel1, com1, com_vel1);
        D3 root_pos0 = GetRootPos(pose0_), root_pos1 = GetRootPos(pose1);
        double pose_err = 0, vel_err = 0, end_eff_err = 0;
        double root_rot_w = joint_weights[0];
        { double th = QuatTheta(QuatDiff(GetRootRot(pose0_), GetRootRot(pose1))); pose_err += root_rot_w * th * th; }      // cKinTree::CalcRootRotErr
        vel_err += root_rot_w * sqnorm(GetRootAngVel(vel1) - GetRootAngVel(vel0_));                                         // cKinTree::CalcRootAngVelErr
        for (int j = 1; j < nj; ++j) {
            const auto& jd = cm->joints[j];
            double w = joint_weights[j], pe = 0, ve = 0;
            if (jd.type == dmh::kSpherical) {  // cKinTree::CalcPoseErr (KinTree.cpp:1319-1352)
                double th = QuatTheta(QuatDiff(pose_quat(pose0_, jd.param_offset), pose_quat(pose1, jd.param_offset)));
                pe = th * th;
            } else for (int k = 0; k < jd.param_size; ++k) { double d = pose1[jd.param_offset + k] - pose0_[jd.param_offset + k]; pe += d * d; }
            for (int k = 0; k < jd.param_size; ++k) { double d = vel1[jd.param_offset + k] - vel0_[jd.param_offset + k]; ve += d * d; }
            pose_err += w * pe; vel_err += w * ve;
            if (jd.is_end_eff) {
                D3 pos0 = JointWorldTransSim(j).t;                   // sim_char.CalcJointPos (SimCharacter.cpp:308-328)
                D3 pos1 = JointWorldTrans(*cm, pose1, j).t;          // cKinTree::CalcJointWorldPos
                double ground_h0 = 0, ground_h1 = origin.y;
                D3 rel0 = pos0 - root_pos0, rel1 = pos1 - root_pos1;
                rel0.y = pos0.y - ground_h0; rel1.y = pos1.y - ground_h1;
                // origin_trans * pos_rel with w == 0: rotation only
                rel0 = ot0.first * rel0; rel1 = ot1.first * rel1;
                end_eff_err += sqnorm(rel1 - rel0);
            }
        }
        double root_ground_h0 = 0, root_ground_h1 = origin.y;
        root_pos0.y -= root_ground_h0; root_pos1.y -= root_ground_h1;
        double root_pos_err = sqnorm(root_pos0 - root_pos1);
        double root_rot_err = QuatDiffTheta(GetRootRot(pose0_), GetRootRot(pose1)); root_rot_err *= root_rot_err;
        double root_vel_err = sqnorm(GetRootVel(vel1) - GetRootVel(vel0_));
        double root_ang_vel_err = sqnorm(GetRootAngVel(vel1) - GetRootAngVel(vel0_));
        double root_err = root_pos_err + 0.1 * root_rot_err + 0.01 * root_vel_err + 0.001 * root_ang_vel_err;
        double com_err = 0.1 * sqnorm(com_vel1 - com_vel0);
        if (dbg) { dbg[0] = pose_err; dbg[1] = vel_err; dbg[2] = end_eff_err; dbg[3] = root_err; dbg[4] = com_err; }
        return pose_w * std::exp(-err_scale * pose_scale * pose_err) + vel_w * std::exp(-err_scale * vel_scale * vel_err) +
               end_eff_w * std::exp(-err_scale * end_eff_scale * end_eff_err) + root_w * std::exp(-err_scale * root_scale * root_err) +
               com_w * std::exp(-err_scale * com_scale * com_err);
    }
    // =================================================================== AMP task scenes (SURVEY 8f rank 2)
    // stateless counter-based uniform in [0,1): identical to dm_policy.cu's u01
    static double U01(uint64_t seed, uint64_t a, uint64_t b) {
        uint64_t z = seed + 0x9E3779B97F4A7C15ull * (a * 2654435761ull + b + 1);
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull; z = (z ^ (z >> 27)) * 0x94D049BB133111EBull; z ^= z >> 31;
        return static_cast<double>(z >> 11) * (1.0 / 9007199254740992.0);
    }
    double Draw() { return U01(task_seed, task_env, task_counter++); }
    double RandDouble(double lo, double hi) { return (lo == hi) ? lo : lo + Draw() * (hi - lo); }   // cRand::RandDouble (util/Rand.cpp:30-41): no draw when min == max
    bool FlipCoin(double p) { return RandDouble(0, 1) < p; }                                         // util/Rand.cpp:137-140
    double RandDoubleNorm(double mean, double stdev) {   // util/Rand.cpp:50-55; Box-Muller on two stream draws (std::normal_distribution is implementation-defined)
        const double u1 = Draw(), u2 = Draw();
        return mean + stdev * std::sqrt(-2.0 * std::log(1.0 - u1)) * std::cos(2.0 * M_PI * u2);
    }
    void TargetTimerReset() { tgt_timer_time = 0; tgt_timer_max = RandDouble(sa.cfg.rand_target_time_min, sa.cfg.rand_target_time_max); }   // cTimer::Reset, uniform (util/Timer.cpp:51-69)
    // cSimCharacter::CalcCOM (SimCharacter.cpp:398-416)
    D3 CalcCOM() const {
        D3 com; double tm = 0;
        for (int b = 0; b < nj; ++b) { com += cm->bodies[b].mass * BodyPos(b); tm += cm->bodies[b].mass; }
        return com / tm;
    }
    // cSceneTargetAMP::SampleRandTargetPos / ResetTargetPos (SceneTargetAMP.cpp:259-279)
    void ResetTargetPos() {
        if (scene_kind == kStrikeAMP) { ResetTargetPosStrike(); return; }
        const D3 root = SimRootPos();
        const double dist = RandDouble(0.0, sa.cfg.max_target_dist);
        const double theta = RandDouble(0.0, 2.0 * M_PI);
        target_pos = D3(root.x + dist * std::cos(theta), 0, root.z + dist * std::sin(theta));
    }
    void SetTargetSpeed(double v) {   // cSceneHeadingAMP::SetTargetSpeed clamps (SceneHeadingAMP.cpp:90-94)
        target_speed = IsHeading() ? std::min(std::max(v, sa.cfg.tar_speed_min), sa.cfg.tar_speed_max) : v;
    }
    // cSceneTargetAMP::ResetTarget / cSceneHeadingAMP::ResetTarget (SceneTargetAMP.cpp:248-251, SceneHeadingAMP.cpp:207-217)
    void ResetTarget() {
        ResetTargetPos();
        if (scene_kind == kStrikeAMP) {   // cSceneStrikeAMP::ResetTarget / ResetTargetHit (SceneStrikeAMP.cpp:300-316,376-383); GetTime() = scene timer
            if (mode == 0 && sa.cfg.init_hit_prob > 0.0) SetTargetHit(FlipCoin(sa.cfg.init_hit_prob));
            target_hit_time = target_hit ? RandDouble(timer_time - sa.cfg.target_hit_reset_time, timer_time) : -1.0;
        }
        if (IsHeading()) {
            const double speed = RandDouble(sa.cfg.tar_speed_min, sa.cfg.tar_speed_max);
            target_heading = 0;
            SetTargetSpeed(speed);
        }
    }
    // cSceneTargetAMP::UpdateTarget / cSceneHeadingAMP::UpdateTarget (SceneTargetAMP.cpp:232-246, SceneHeadingAMP.cpp:192-205);
    // mEnableRandTargetPos stays true in both scenes (set by the cSceneTargetAMP constructor), mEnableTargetPos false, mEnableRandSpeed true
    void UpdateTarget(double dt) {
        tgt_timer_time += dt;
        const bool timer_end = tgt_timer_time >= tgt_timer_max;
        if (scene_kind == kStrikeAMP) {   // CheckTargetReset is false here (:385-388): the target only moves at a reset; UpdateTarget (:289-298)
            if (!target_hit) SetTargetHit(CheckTargetHit());
            return;
        }
        if (timer_end) ResetTargetPos();
        if (IsHeading() && timer_end) {
            // UpdateTargetHeading (SceneHeadingAMP.cpp:148-180)
            double delta_heading;
            if (FlipCoin(sa.cfg.sharp_turn_prob)) delta_heading = RandDouble(-M_PI, M_PI);
            else delta_heading = RandDoubleNorm(0, sa.cfg.max_heading_turn_rate);
            target_heading += delta_heading;
            // UpdateTargetSpeed (SceneHeadingAMP.cpp:182-190)
            if (FlipCoin(sa.cfg.speed_change_prob)) SetTargetSpeed(RandDouble(sa.cfg.tar_speed_min, sa.cfg.tar_speed_max));
        }
    }
    int GoalSize() const { return (scene_kind == kHeadingGetup || scene_kind == kStrikeAMP) ? 4 : (IsTask() ? 3 : 0); }   // + getup phase (SceneHeadingAMPGetup.cpp:135-140)   // SceneTargetAMP.cpp:217-220, SceneHeadingAMP.cpp:131-134; 0 otherwise (RLSceneSimChar.cpp:88-91)
    // cSceneTargetAMP::RecordGoal (SceneTargetAMP.cpp:185-215) / cSceneHeadingAMP::RecordGoal (SceneHeadingAMP.cpp:136-151)
    void RecordGoal(double* out) const {
        if (scene_kind == kTargetAMP) {
            const D3 root = SimRootPos();
            D3 rel = target_pos - root; rel.y = 0;
            const double dist = norm(rel);
            if (dist > 0.0001) {
                const DM3 Rh = RotateMatAxis(D3(0, 1, 0), -CalcHeading(GetRootRot(pose)));   // cKinTree::BuildOriginTrans applied to a direction (w = 0)
                rel = (Rh * rel) / dist;
            } else rel = D3(1, 0, 0);
            out[0] = rel.x; out[1] = rel.z; out[2] = dist;
        } else if (scene_kind == kStrikeAMP) {   // cSceneStrikeAMP::RecordGoal (:407-430): target in the origin frame (translation included) + hit phase
            const D3 root = SimRootPos();
            const DM3 Rh = RotateMatAxis(D3(0, 1, 0), -CalcHeading(GetRootRot(pose)));
            const D3 rp = GetRootPos(pose);
            const D3 loc = Rh * (target_pos - D3(rp.x, 0, rp.z));   // cKinTree::BuildOriginTrans: origin = root x, z on the ground
            out[0] = loc.x; out[1] = loc.y; out[2] = loc.z; out[3] = CalcHitPhase();
            (void)root;
        } else if (IsHeading()) {
            const double th = target_heading - CalcHeading(GetRootRot(pose));
            out[0] = std::cos(th); out[1] = -std::sin(th); out[2] = target_speed;
            if (scene_kind == kHeadingGetup) out[3] = std::min(std::max(1.0 - getup_timer_time / getup_time, 0.0), 1.0);   // CalcGetupPhase (:289-294)
        }
    }
    bool CheckTarDistFail() const {   // SceneTargetAMP.cpp:281-292; always false in the heading scene (SceneHeadingAMP.cpp:219-222)
        if (scene_kind != kTargetAMP && scene_kind != kStrikeAMP) return false;
        D3 d = SimRootPos() - target_pos; d.y = 0;
        return sqnorm(d) > sa.cfg.tar_fail_dist * sa.cfg.tar_fail_dist;
    }
    bool CheckTargetSucc() const {   // SceneTargetAMP.cpp:171-183
        D3 d = target_pos - SimRootPos(); d.y = 0;
        return norm(d) < sa.cfg.target_succ_dist;
    }
    // cSceneTargetAMP::CalcReward (SceneTargetAMP.cpp:3-80)
    double CalcRewardTarget() const {
        const double pos_reward_w = 0.6, vel_reward_w = 0.4;
        if (CheckTarDistFail() || HasFallen()) return 0.0;
        const double tar_speed = target_speed;
        const double vel_err_scale = 4 / (tar_speed * tar_speed);
        D3 root_tar_delta = target_pos - SimRootPos(); root_tar_delta.y = 0;
        const double root_tar_dist_sq = sqnorm(root_tar_delta);
        const double pos_reward = std::exp(-sa.cfg.pos_reward_scale * root_tar_dist_sq);
        double vel_reward = 0;
        if (root_tar_dist_sq < sa.cfg.target_succ_dist * sa.cfg.target_succ_dist) vel_reward = 1.0;
        else {
            const double step_dur = ctrl_time - prev_action_time;
            const D3 com = CalcCOM();
            D3 com_tar_delta = target_pos - com; com_tar_delta.y = 0;
            const double com_tar_dist = norm(com_tar_delta);
            D3 com_tar_dir;
            if (com_tar_dist > 0.0001) com_tar_dir = com_tar_delta / com_tar_dist;
            const double avg_vel = dot(com_tar_dir, com - prev_action_com) / step_dur;
            double vel_err = tar_speed - avg_vel;
            if (avg_vel < 0) vel_reward = 0.0;
            else {
                if (sa.cfg.enable_min_tar_vel) vel_err = std::max(vel_err, 0.0);
                vel_reward = std::exp(-vel_err_scale * vel_err * vel_err);
            }
        }
        return pos_reward_w * pos_reward + vel_reward_w * vel_reward;
    }
    // cSceneHeadingAMP::CalcReward (SceneHeadingAMP.cpp:3-48)
    double CalcRewardHeading() const {
        if (HasFallen()) return 0.0;
        const D3 com = CalcCOM();
        const D3 tar_dir(std::cos(target_heading), 0, -std::sin(target_heading));
        const double step_dur = ctrl_time - prev_action_time;
        D3 avg_vel = (com - prev_action_com) / step_dur; avg_vel.y = 0;
        const double avg_speed = dot(tar_dir, avg_vel);
        double vel_reward = 0;
        if (avg_speed > 0.0) {
            double vel_err = target_speed - avg_speed;
            if (sa.cfg.enable_min_tar_vel) vel_err = std::max(vel_err, 0.0);
            vel_reward = std::exp(-sa.cfg.vel_reward_scale * vel_err * vel_err);
        }
        return vel_reward;
    }

    // ------------------------------------------------------------------- cSceneStrikeAMP (scenes/SceneStrikeAMP.cpp)
    void SetTargetHit(bool hit) { if (!target_hit && hit) target_hit_time = timer_time; target_hit = hit; }   // :246-255
    // ResetTargetPos / ResetTargetPosFar / ResetTargetPosNear (:318-374)
    void ResetTargetPosStrike() {
        const D3 root = SimRootPos();
        const dmh::V3 &mn = sa.cfg.target_min, &mx = sa.cfg.target_max;
        double theta, h, dist;
        if (FlipCoin(sa.cfg.tar_far_prob)) { theta = RandDouble(-M_PI, M_PI); h = RandDouble(mn.y, mx.y); dist = RandDouble(mn.z, sa.cfg.max_target_dist); }
        else { theta = RandDouble(mn.x, mx.x); h = RandDouble(mn.y, mx.y); dist = RandDouble(mn.z, mx.z); }
        SetTargetHit(false);
        target_pos = D3(root.x + dist * std::cos(theta), h, root.z - dist * std::sin(theta));   // flat ground at 0
    }
    // CheckTargetHit (:440-481): a strike body inside the target sphere, moving towards the target (seen from the root) fast enough
    bool CheckTargetHit() const {
        D3 d = target_pos - SimRootPos(); d.y = 0;
        const double n = norm(d);
        D3 dir; if (n > 1e-5) dir = d / n;
        for (int b : sa.cfg.strike_bodies) {
            if (sqnorm(target_pos - BodyPos(b)) < sa.cfg.target_radius * sa.cfg.target_radius) {
                const double speed = dot(dir, link_lin_vel[b]);
                if (speed >= sa.cfg.hit_tar_speed || sa.cfg.hit_tar_speed == 0.0) return true;
            }
        }
        return false;
    }
    bool CheckTarContactFail() const {   // :489-508
        for (int b : sa.cfg.fail_tar_contact_bodies) if (sqnorm(target_pos - BodyPos(b)) < sa.cfg.target_radius * sa.cfg.target_radius) return true;
        return false;
    }
    bool CheckTarHitSucc() const { return target_hit && (timer_time - target_hit_time) >= sa.cfg.target_hit_reset_time; }   // :510-524
    double CalcHitPhase() const {   // :390-401
        if (!target_hit) return 0.0;
        return std::min(std::max((timer_time - target_hit_time) / sa.cfg.target_hit_reset_time, 0.0), 1.0);
    }
    // CalcReward / CalcRewardTrain / CalcRewardTest / CalcRewardTargetNear / CalcRewardTargetFar (:9-190)
    double CalcRewardStrike() const {
        const double far_w = 0.3, near_w = 0.3, hit_w = 0.4;
        if (mode == 1) return (IsEpisodeEnd() && CheckTerminate() == 2) ? timer_max - timer_time : 0.0;
        const D3 root = SimRootPos();
        D3 trd = target_pos - root; trd.y = 0;
        const double dist_sq = sqnorm(trd), near_dist = sa.cfg.tar_near_dist;
        if (target_hit) return far_w + near_w + hit_w;
        if (dist_sq < near_dist * near_dist) {
            // near: best strike body, 0.2 distance term + 0.8 squared normalised speed towards the target
            const double n = std::sqrt(dist_sq);
            D3 dir; if (n > 1e-5) dir = trd / n;
            double r = 0.0;
            for (int b : sa.cfg.strike_bodies) {
                const double dr = std::exp(-sa.cfg.tar_reward_scale * sqnorm(target_pos - BodyPos(b)));
                double vr = std::min(std::max(dot(dir, link_lin_vel[b]) / sa.cfg.hit_tar_speed, 0.0), 1.0);
                vr *= vr;
                r = std::max(r, 0.2 * dr + 0.8 * vr);
            }
            return far_w + near_w * r;
        }
        // far: like the target scene, but the position term measures the distance to the near radius
        double r = 0.0;
        if (!HasFallen()) {
            const double tar_speed = target_speed, vel_err_scale = 4 / (tar_speed * tar_speed);
            const double root_tar_dist = std::sqrt(dist_sq);
            const double root_dist_err = std::max(root_tar_dist - near_dist, 0.0);
            const double pos_reward = std::exp(-sa.cfg.pos_reward_scale * root_dist_err * root_dist_err);
            double vel_reward = 0;
            if (root_tar_dist < near_dist) vel_reward = 1.0;
            else {
                const double step_dur = ctrl_time - prev_action_time;
                const D3 com = CalcCOM();
                D3 ctd = target_pos - com; ctd.y = 0;
                const double cd = norm(ctd);
                D3 cdir; if (cd > 0.0001) cdir = ctd / cd;
                const double avg_vel = dot(cdir, com - prev_action_com) / step_dur;
                double vel_err = tar_speed - avg_vel;
                if (avg_vel < 0) vel_reward = 0.0;
                else { if (sa.cfg.enable_min_tar_vel) vel_err = std::max(vel_err, 0.0); vel_reward = std::exp(-vel_err_scale * vel_err * vel_err); }
            }
            r = 0.7 * pos_reward + 0.3 * vel_reward;
        }
        return far_w * r;
    }

    // cRLSceneSimChar::CheckTerminate + cSceneImitate::CheckTerminate (RLSceneSimChar.cpp:187-197; SceneImitate.cpp:193-205)
    int CheckTerminate() const {
        bool fail = sa.cfg.enable_fall_end && HasFallen();
        // the AMP scenes use cRLSceneSimChar::CheckTerminate alone (SceneImitateAMP.cpp:185-189): no motion-over failure there
        if (!fail && scene_kind == kImitate && !Mot().loop && kin_time >= Mot().duration()) fail = true;
        if (!fail && scene_kind == kTargetAMP && CheckTarDistFail()) fail = true;   // cSceneTargetAMP::CheckTerminate (SceneTargetAMP.cpp:294-319)
        if (!fail && scene_kind == kStrikeAMP) {   // cSceneStrikeAMP::CheckTerminateTarget (:526-546): distance, forbidden bodies at the target, then success (2)
            if (CheckTarDistFail() || CheckTarContactFail()) fail = true;
            else if (CheckTarHitSucc()) return 2;
        }
        return fail ? 1 : 0;
    }
    bool IsEpisodeEnd() const { return timer_time >= timer_max || CheckTerminate() != 0; }  // RLScene.cpp:36-50
    bool CheckValidEpisode() const {  // cSimCharacter::HasVelExploded (SimCharacter.cpp:571-586)
        for (int b = 0; b < nj; ++b) {
            const D3& v = link_lin_vel[b]; const D3& w = link_ang_vel[b];
            double mx = std::max(std::max(std::max(std::fabs(v.x), std::fabs(v.y)), std::fabs(v.z)), std::max(std::max(std::fabs(w.x), std::fabs(w.y)), std::fabs(w.z)));
            if (mx > 100.0) return false;
        }
        return true;
    }
    // action offset / scale / bounds (CtCtrlUtil.cpp:255-286,357-398,464-474; CtController.cpp:71-101,229-262)
    void ActionStatics(double* off, double* scl, double* bmin, double* bmax) const {
        for (int j = 1; j < nj; ++j) {
            const auto& jd = cm->joints[j];
            if (jd.type == dmh::kSpherical) {
                for (int k = 0; k < 3; ++k) { off[ctrl_off[j] + k] = 0; scl[ctrl_off[j] + k] = 2.0 / (2.0 * M_PI); bmin[ctrl_off[j] + k] = -2.0 * M_PI; bmax[ctrl_off[j] + k] = 2.0 * M_PI; }
            } else if (jd.type == dmh::kRevolute) {
                double lo = jd.lim_low[0], hi = jd.lim_high[0];
                if (!(hi >= lo)) { lo = -M_PI; hi = M_PI; }
                off[ctrl_off[j]] = -0.5 * (hi + lo); scl[ctrl_off[j]] = 0.5 / (hi - lo);
                double mean = 0.5 * (hi + lo), delta = hi - lo;
                bmin[ctrl_off[j]] = mean - 2 * delta; bmax[ctrl_off[j]] = mean + 2 * delta;
            }
        }
    }

    // =================================================================== raw state snapshot (test hook shared with the CUDA path)
    // layout documented in include/deepmimic_b200.h (dm_snapshot_size)
    int SnapshotSize() const { return 29 + 59 * nj; }
    void GetSnapshot(double* s) const {
        std::fill(s, s + SnapshotSize(), 0.0);
        s[0] = mb.basePos.x; s[1] = mb.basePos.y; s[2] = mb.basePos.z;
        s[3] = mb.baseQuat.x; s[4] = mb.baseQuat.y; s[5] = mb.baseQuat.z; s[6] = mb.baseQuat.w;
        for (int k = 0; k < 6; ++k) s[7 + k] = mb.realBuf[k];
        for (int j = 0; j < nj; ++j) {
            for (int k = 0; k < 4; ++k) s[13 + 4 * j + k] = mb.links[j].jointPos[k];
            const float* qd = mb.jointVel(j);
            for (int k = 0; k < mb.links[j].dofCount; ++k) s[13 + 4 * nj + 3 * j + k] = qd[k];
            const BtManifold& m = mb.links[j].manifold;
            for (int c = 0; c < m.n; ++c) {
                double* o = s + 13 + 7 * nj + (j * 4 + c) * 12;
                const BtManifoldPoint& p = m.pt[c];
                o[0] = 1; o[1] = p.localPointA.x; o[2] = p.localPointA.y; o[3] = p.localPointA.z; o[4] = p.localPointB.x; o[5] = p.localPointB.y; o[6] = p.localPointB.z;
                o[7] = p.appliedImpulse; o[8] = p.appliedImpulseLateral1; o[9] = p.appliedImpulseLateral2; o[10] = p.distance1; o[11] = p.lifeTime;
            }
        }
        double* q = s + 13 + 55 * nj;
        q[0] = kin_time; q[1] = origin.x; q[2] = origin.y; q[3] = origin.z; q[4] = origin_rot.w; q[5] = origin_rot.x; q[6] = origin_rot.y; q[7] = origin_rot.z;
        q[8] = ctrl_time; q[9] = init_time_offset; q[10] = prev_action_time; q[11] = need_new_action ? 1 : 0; q[12] = timer_time; q[13] = timer_max;
        double* t = q + 16;
        for (int j = 0; j < nj; ++j) for (int k = 0; k < 4; ++k) t[4 * j + k] = tar_theta[j][k];
    }
    void SetSnapshot(const double* s) {
        mb.basePos = F3(static_cast<float>(s[0]), static_cast<float>(s[1]), static_cast<float>(s[2]));
        mb.baseQuat = FQ(static_cast<float>(s[3]), static_cast<float>(s[4]), static_cast<float>(s[5]), static_cast<float>(s[6]));
        for (int k = 0; k < 6; ++k) mb.realBuf[k] = static_cast<float>(s[7 + k]);
        for (int j = 0; j < nj; ++j) {
            BtLink& L = mb.links[j];
            if (L.dofCount > 0) for (int k = 0; k < 4; ++k) L.jointPos[k] = static_cast<float>(s[13 + 4 * j + k]);
            float* qd = mb.jointVel(j);
            for (int k = 0; k < L.dofCount; ++k) qd[k] = static_cast<float>(s[13 + 4 * nj + 3 * j + k]);
            L.updateCache();
            BtManifold& m = L.manifold;
            m.n = 0;
            for (int c = 0; c < 4; ++c) {
                const double* o = s + 13 + 7 * nj + (j * 4 + c) * 12;
                if (o[0] == 0) break;
                BtManifoldPoint& p = m.pt[m.n++];
                p.localPointA = F3(static_cast<float>(o[1]), static_cast<float>(o[2]), static_cast<float>(o[3]));
                p.localPointB = F3(static_cast<float>(o[4]), static_cast<float>(o[5]), static_cast<float>(o[6]));
                p.appliedImpulse = static_cast<float>(o[7]); p.appliedImpulseLateral1 = static_cast<float>(o[8]); p.appliedImpulseLateral2 = static_cast<float>(o[9]);
                p.distance1 = static_cast<float>(o[10]); p.lifeTime = static_cast<int>(o[11]);
            }
        }
        mb.updateCollisionObjectWorldTransforms();
        snap_frames.assign(12 * nj, 0.0f);
        for (int j = 0; j < nj; ++j) {
            const BtLink& L = mb.links[j];
            for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) snap_frames[12 * j + 3 * r + c] = L.worldBasis.m[r][c];
            snap_frames[12 * j + 9] = L.worldPos.x; snap_frames[12 * j + 10] = L.worldPos.y; snap_frames[12 * j + 11] = L.worldPos.z;
        }
        const double* q = s + 13 + 55 * nj;
        kin_time = q[0]; origin = D3(q[1], q[2], q[3]); origin_rot = DQ(q[4], q[5], q[6], q[7]);
        ctrl_time = q[8]; init_time_offset = q[9]; prev_action_time = q[10]; need_new_action = q[11] != 0; timer_time = q[12]; timer_max = q[13];
        const double* t = q + 16;
        for (int j = 0; j < nj; ++j) for (int k = 0; k < 4; ++k) tar_theta[j][k] = t[4 * j + k];
        KinPose();
        UpdateLinkVel();
        BuildPoseVel();
    }
};

}  // namespace orc

// ======================================================================= C API (ctypes; tests/bench only)
using orc::Oracle;
static std::string g_err;
extern "C" {

void* dmo_create(const char* asset_root, int argc, const char** argv) {
    try {
        std::vector<std::string> args(argv, argv + argc);
        dmh::ArgParser ap;
        ap.LoadArgs(args);
        std::string arg_file;
        if (ap.ParseString("arg_file", arg_file)) {
            if (!ap.LoadFile(dmh::resolve_path(asset_root ? asset_root : "", arg_file))) throw std::runtime_error("Failed to load args from: " + arg_file);
        }
        auto o = std::make_unique<Oracle>();
        o->Init(dmh::load_scene_assets(ap, asset_root ? asset_root : ""));
        return o.release();
    } catch (const std::exception& e) {
        g_err = e.what();
        std::fprintf(stderr, "[dm_oracle] %s\n", e.what());
        return nullptr;
    }
}
const char* dmo_last_error() { return g_err.c_str(); }
void dmo_destroy(void* h) { delete static_cast<Oracle*>(h); }
// out[0..7] = num_joints, pose_dim, bullet_dofs(6+n), state_size, action_size, goal_size, snapshot_size, num_frames
void dmo_get_dims(void* h, int* out) {
    Oracle* o = static_cast<Oracle*>(h);
    out[0] = o->nj; out[1] = o->ndof; out[2] = 6 + o->mb.numDofs; out[3] = o->StateSize(); out[4] = o->action_size; out[5] = o->GoalSize(); out[6] = o->SnapshotSize(); out[7] = o->sa.motion.num_frames;
}
// test hook mirroring dm_get_link_table (same 24-double rows) from the oracle's own multibody: mass, Bullet inertia, cRBDUtil moment of inertia
// (diagonal of BuildMomentInertia), dVector, eVector, zeroRotParentToThis (x,y,z,w), axis, half extents, breaking threshold
void dmo_link_table(void* h, double* out) {
    Oracle* o = static_cast<Oracle*>(h);
    for (int j = 0; j < o->nj; ++j) {
        const orc::BtLink& L = o->mb.links[j];
        double* q = out + 24 * j;
        q[0] = L.mass;
        q[1] = L.inertia.x; q[2] = L.inertia.y; q[3] = L.inertia.z;
        const orc::SpMat I = orc::BuildMomentInertia(*o->cm, j);
        q[4] = I.m[0][0]; q[5] = I.m[1][1]; q[6] = I.m[2][2];
        q[7] = L.dVector.x; q[8] = L.dVector.y; q[9] = L.dVector.z; q[10] = L.eVector.x; q[11] = L.eVector.y; q[12] = L.eVector.z;
        q[13] = L.zeroRotParentToThis.x; q[14] = L.zeroRotParentToThis.y; q[15] = L.zeroRotParentToThis.z; q[16] = L.zeroRotParentToThis.w;
        q[17] = L.axisTop[0].x; q[18] = L.axisTop[0].y; q[19] = L.axisTop[0].z;
        q[20] = L.halfExtents.x; q[21] = L.halfExtents.y; q[22] = L.halfExtents.z;
        q[23] = L.manifold.breakingThreshold;
    }
}
double dmo_motion_duration(void* h) { return static_cast<Oracle*>(h)->Mot().duration(); }
void dmo_set_mode(void* h, int mode) { static_cast<Oracle*>(h)->mode = mode; }
void dmo_reset(void* h, double kin_time, double rand_theta, double max_time) { static_cast<Oracle*>(h)->Reset(kin_time, rand_theta, max_time); }
void dmo_reset_clip(void* h, int clip, double kin_time, double rand_theta, double max_time) { static_cast<Oracle*>(h)->Reset(kin_time, rand_theta, max_time, clip); }
// clip dataset of --kin_ctrl clips: count; per clip duration / weight / cdf / loop flag; active clip; cClipsController::SelectNewMotion on a given uniform draw
int dmo_num_clips(void* h) { return static_cast<int>(static_cast<Oracle*>(h)->sa.clips.size()); }
void dmo_clip_table(void* h, double* dur, double* weight, double* cdf, int* loop) {
    Oracle* o = static_cast<Oracle*>(h);
    for (size_t c = 0; c < o->sa.clips.size(); ++c) { dur[c] = o->sa.clips[c].duration(); weight[c] = o->sa.clip_weights[c]; cdf[c] = o->sa.clip_cdf[c]; loop[c] = o->sa.clips[c].loop ? 1 : 0; }
}
int dmo_current_clip(void* h) { return static_cast<Oracle*>(h)->cur_clip; }
int dmo_select_clip(void* h, double u01) { return static_cast<Oracle*>(h)->sa.select_clip(u01); }
// AMP task scenes
void dmo_set_task_stream(void* h, unsigned long long seed, unsigned long long env, unsigned long long counter) { Oracle* o = static_cast<Oracle*>(h); o->task_seed = seed; o->task_env = env; o->task_counter = counter; }
unsigned long long dmo_task_counter(void* h) { return static_cast<Oracle*>(h)->task_counter; }
double dmo_u01(unsigned long long seed, unsigned long long a, unsigned long long b) { return Oracle::U01(seed, a, b); }
void dmo_record_goal(void* h, double* out) { static_cast<Oracle*>(h)->RecordGoal(out); }
// out[0..7] = target_pos xyz, target_speed, target_heading, target timer time, target timer max, prev_action_com x (then y, z in out[8], out[9])
void dmo_get_task_state(void* h, double* out) {
    Oracle* o = static_cast<Oracle*>(h);
    out[0] = o->target_pos.x; out[1] = o->target_pos.y; out[2] = o->target_pos.z; out[3] = o->target_speed; out[4] = o->target_heading;
    out[5] = o->tgt_timer_time; out[6] = o->tgt_timer_max; out[7] = o->prev_action_com.x; out[8] = o->prev_action_com.y; out[9] = o->prev_action_com.z;
}
void dmo_set_task_state(void* h, const double* in) {
    Oracle* o = static_cast<Oracle*>(h);
    o->target_pos = orc::D3(in[0], in[1], in[2]); o->target_speed = in[3]; o->target_heading = in[4]; o->tgt_timer_time = in[5]; o->tgt_timer_max = in[6];
    o->prev_action_com = orc::D3(in[7], in[8], in[9]);
}
// heading_amp_getup: out[0] = get-up timer, out[1] = get-up time (its end), out[2] = getting up (0 / 1), out[3] = contact fall ignoring the get-up override
void dmo_get_getup_state(void* h, double* out) {
    Oracle* o = static_cast<Oracle*>(h);
    out[0] = o->getup_timer_time; out[1] = o->getup_time; out[2] = o->CheckGettingUp() ? 1 : 0; out[3] = o->ContactFall() ? 1 : 0;
}
void dmo_set_getup_timer(void* h, double t) { static_cast<Oracle*>(h)->getup_timer_time = t; }
// strike_amp: out[0] = target hit (0 / 1), out[1] = hit time, out[2] = hit phase, out[3] = target height
void dmo_get_strike_state(void* h, double* out) { Oracle* o = static_cast<Oracle*>(h); out[0] = o->target_hit ? 1 : 0; out[1] = o->target_hit_time; out[2] = o->CalcHitPhase(); out[3] = o->target_pos.y; }
void dmo_set_strike_state(void* h, int hit, double hit_time) { Oracle* o = static_cast<Oracle*>(h); o->target_hit = hit != 0; o->target_hit_time = hit_time; }
int dmo_check_target_succ(void* h) { return static_cast<Oracle*>(h)->CheckTargetSucc() ? 1 : 0; }
int dmo_enable_amp_task_reward(void* h) { return static_cast<Oracle*>(h)->IsTask() ? 1 : 0; }   // SceneTargetAMP.cpp:222-225
void dmo_calc_com(void* h, double* out) { orc::D3 c = static_cast<Oracle*>(h)->CalcCOM(); out[0] = c.x; out[1] = c.y; out[2] = c.z; }
void dmo_update(void* h, double dt) { static_cast<Oracle*>(h)->Update(dt); }
// test hook: a timed push, an external force for one Update.  cWorld::Update keeps applied forces through stepSimulation until its final
// clearForces, and nothing in cSceneSimChar::Update before stepSimulation touches them, so the force is added to the body's link (Bullet's
// link frame sits at the body's COM) right before the oracle's own Update and acts in both of its sub-steps.
// One Update(dt), with force (world axes, unscaled N) times the world scale on `body` when body >= 0 and the timer value at the update's start t
// satisfies start <= t < start + duration (the scale rule of gravity: the unscaled character sees F / m).
void dmo_update_pushed(void* h, double dt, int body, const double* force, double start, double duration) {
    orc::Oracle* o = static_cast<orc::Oracle*>(h);
    const double t = o->timer_time;
    if (body >= 0 && start <= t && t < start + duration)
        o->mb.links[body].appliedForce += orc::F3(static_cast<float>(force[0] * o->scale), static_cast<float>(force[1] * o->scale), static_cast<float>(force[2] * o->scale));
    o->Update(dt);
}
// test hook: the contact friction coefficient Bullet's solver uses for every contact (the reference's link friction times the ground's).
// Masses, gains and torque limits need no hook: the tests edit them in a copy of the asset files.
void dmo_set_contact_friction(void* h, double mu) { static_cast<orc::Oracle*>(h)->friction = mu; }
void dmo_set_action(void* h, const double* a) { static_cast<Oracle*>(h)->SetAction(a); }
void dmo_record_state(void* h, double* out) { static_cast<Oracle*>(h)->RecordState(out); }
int dmo_amp_obs_size(void* h) { return static_cast<Oracle*>(h)->AmpObsSize(); }
void dmo_record_amp_obs_agent(void* h, double* out) { static_cast<Oracle*>(h)->RecordAMPObsAgent(out); }
// test hook: the AMP history := the current pose / vel, as the first update after a new action sets it (cSceneImitateAMP::UpdateHist)
void dmo_update_hist(void* h) { static_cast<Oracle*>(h)->UpdateHist(); }
void dmo_record_amp_obs_expert(void* h, double kin_time, double* out) { static_cast<Oracle*>(h)->RecordAMPObsExpert(-1, kin_time, out); }
void dmo_record_amp_obs_expert_clip(void* h, int clip, double kin_time, double* out) { static_cast<Oracle*>(h)->RecordAMPObsExpert(clip, kin_time, out); }
double dmo_calc_reward(void* h) { return static_cast<Oracle*>(h)->CalcReward(); }
double dmo_calc_reward_imitate(void* h) { return static_cast<Oracle*>(h)->CalcReward(nullptr, true); }
double dmo_calc_reward_terms(void* h, double* errs) { return static_cast<Oracle*>(h)->CalcReward(errs); }
int dmo_need_new_action(void* h) { return static_cast<Oracle*>(h)->need_new_action ? 1 : 0; }
int dmo_is_episode_end(void* h) { return static_cast<Oracle*>(h)->IsEpisodeEnd() ? 1 : 0; }
int dmo_check_terminate(void* h) { return static_cast<Oracle*>(h)->CheckTerminate(); }
int dmo_check_valid_episode(void* h) { return static_cast<Oracle*>(h)->CheckValidEpisode() ? 1 : 0; }
int dmo_has_fallen(void* h) { return static_cast<Oracle*>(h)->HasFallen() ? 1 : 0; }
double dmo_get_time(void* h) { return static_cast<Oracle*>(h)->timer_time; }
void dmo_get_pose(void* h, double* pose, double* vel) { Oracle* o = static_cast<Oracle*>(h); std::copy(o->pose.begin(), o->pose.end(), pose); std::copy(o->vel.begin(), o->vel.end(), vel); }
void dmo_get_kin_pose(void* h, double* pose, double* vel) { Oracle* o = static_cast<Oracle*>(h); std::copy(o->kin_pose.begin(), o->kin_pose.end(), pose); std::copy(o->kin_vel.begin(), o->kin_vel.end(), vel); }
void dmo_set_pose_vel(void* h, const double* pose, const double* vel) { Oracle* o = static_cast<Oracle*>(h); orc::VecD p(pose, pose + o->ndof), v(vel, vel + o->ndof); o->SetPose(p); o->SetVel(v); }
void dmo_get_snapshot(void* h, double* s) { static_cast<Oracle*>(h)->GetSnapshot(s); }
void dmo_set_snapshot(void* h, const double* s) { static_cast<Oracle*>(h)->SetSnapshot(s); }
void dmo_action_statics(void* h, double* off, double* scl, double* bmin, double* bmax) { static_cast<Oracle*>(h)->ActionStatics(off, scl, bmin, bmax); }
// KAT hooks: DeepMimic-model mass matrix / bias force at the current pose, SPD torque, Bullet-model ABA acceleration
void dmo_rbd_mass_bias(void* h, double* M, double* C) { Oracle* o = static_cast<Oracle*>(h); o->rbd.Update(o->pose, o->vel); std::copy(o->rbd.M.begin(), o->rbd.M.end(), M); std::copy(o->rbd.C.begin(), o->rbd.C.end(), C); }
void dmo_spd_tau(void* h, double dt, double* tau) { Oracle* o = static_cast<Oracle*>(h); orc::VecD t(o->ndof, 0.0); o->rbd.Update(o->pose, o->vel); o->CalcControlForces(dt, t); std::copy(t.begin(), t.end(), tau); }
void dmo_inv_dyna(void* h, const double* acc, double* tau) { Oracle* o = static_cast<Oracle*>(h); orc::VecD a(acc, acc + o->ndof), t; o->rbd.Update(o->pose, o->vel); o->rbd.SolveInvDyna(a, t); std::copy(t.begin(), t.end(), tau); }
// one contact-free Bullet ABA evaluation with the given generalised joint torques (Bullet dof order, scaled units): returns dv/dt
void dmo_bullet_aba(void* h, const float* joint_tau, int with_gravity, float* out_acc) {
    Oracle* o = static_cast<Oracle*>(h);
    orc::BtMultiBody mb = o->mb;  // copy
    for (auto& L : mb.links) { L.appliedForce = with_gravity ? L.mass * mb.gravity : orc::F3(); for (int d = 0; d < L.dofCount; ++d) L.jointTorque[d] = joint_tau[L.dofOffset + d]; }
    std::vector<float> before = mb.realBuf;
    mb.maxCoordinateVelocity = 1e30f;
    mb.computeAccelerationsABA(1.0f);
    for (size_t k = 0; k < before.size(); ++k) out_acc[k] = mb.realBuf[k] - before[k];
}
// debug taps of the last Update: out = [after ABA (ndofs) | after PGS (ndofs) | lambdas (64)]
void dmo_debug_taps(void* h, float* out) {
    Oracle* o = static_cast<Oracle*>(h); int n = 6 + o->mb.numDofs;
    for (int k = 0; k < n; ++k) { out[k] = k < (int)o->mb.dbg_after_aba.size() ? o->mb.dbg_after_aba[k] : 0; out[n + k] = k < (int)o->mb.dbg_after_pgs.size() ? o->mb.dbg_after_pgs[k] : 0; }
    for (int k = 0; k < 64; ++k) out[2 * n + k] = k < (int)o->mb.dbg_lambda.size() ? o->mb.dbg_lambda[k] : 0;
}
void dmo_debug_taps1(void* h, float* out) {
    Oracle* o = static_cast<Oracle*>(h); int n = 6 + o->mb.numDofs;
    for (int k = 0; k < n; ++k) { out[k] = k < (int)o->mb.dbg_after_aba1.size() ? o->mb.dbg_after_aba1[k] : 0; out[n + k] = k < (int)o->mb.dbg_after_pgs1.size() ? o->mb.dbg_after_pgs1[k] : 0; }
    for (int k = 0; k < 64; ++k) out[2 * n + k] = k < (int)o->mb.dbg_lambda1.size() ? o->mb.dbg_lambda1[k] : 0;
}
// constraint-solve branches of each Bullet sub-step of the last Update: 7 ints per sub-step (limit rows, contact points, clamp in the
// unconstrained update, clamp after PGS, limit rows at the impulse cap, friction rows skipped in the last sweep, limit rows past the
// split-impulse threshold), at most max_substeps sub-steps; returns the number of sub-steps
int dmo_last_rows(void* h, int* out, int max_substeps) {
    const auto& rows = static_cast<Oracle*>(h)->mb.dbg_rows;
    const int n = std::min(static_cast<int>(rows.size()), max_substeps);
    for (int s = 0; s < n; ++s) {
        const auto& t = rows[s];
        const int v[7] = {t.limits, t.points, t.clampAba, t.clampPgs, t.limitsAtUpper, t.frictionSkipped, t.limitsDeep};
        std::copy(v, v + 7, out + 7 * s);
    }
    return n;
}
// link-plane collision branches of each Bullet sub-step of the last Update: 6 ints per (sub-step, link) (event: 0 none / 1 add / 2 replace
// nearest / 3 full-cache insert, slot written, deepest slot kept by sortCachedPoints or -1, mask of slots removed by distance, mask removed
// by lateral drift, points after the refresh), at most max_substeps sub-steps; returns the number of sub-steps
int dmo_last_contacts(void* h, int* out, int max_substeps) {
    const auto& taps = static_cast<Oracle*>(h)->mb.dbg_contacts;
    const int n = std::min(static_cast<int>(taps.size()), max_substeps);
    for (int s = 0; s < n; ++s)
        for (size_t i = 0; i < taps[s].size(); ++i) {
            const auto& t = taps[s][i];
            const int v[6] = {t.event, t.slot, t.deepest, t.rmDist, t.rmDrift, t.count};
            std::copy(v, v + 6, out + 6 * (s * taps[s].size() + i));
        }
    return n;
}
// each link's collider frame as of the last set_snapshot: 12 doubles per link (worldBasis row-major, worldPos), scaled units
void dmo_collider_frames(void* h, double* out) {
    const auto& f = static_cast<Oracle*>(h)->snap_frames;
    std::copy(f.begin(), f.end(), out);
}
void dmo_kin_frame(void* h, double time, double* pose, double* vel) { Oracle* o = static_cast<Oracle*>(h); orc::VecD p, v; o->KinCalcPose(time, p); o->KinCalcVel(time, v); std::copy(p.begin(), p.end(), pose); std::copy(v.begin(), v.end(), vel); }
void dmo_body_state(void* h, double* pos, double* rot, double* linvel, double* angvel) {
    Oracle* o = static_cast<Oracle*>(h);
    for (int b = 0; b < o->nj; ++b) {
        orc::D3 p = o->BodyPos(b); orc::DQ q = o->BodyRot(b);
        pos[3 * b] = p.x; pos[3 * b + 1] = p.y; pos[3 * b + 2] = p.z; rot[4 * b] = q.w; rot[4 * b + 1] = q.x; rot[4 * b + 2] = q.y; rot[4 * b + 3] = q.z;
        linvel[3 * b] = o->link_lin_vel[b].x; linvel[3 * b + 1] = o->link_lin_vel[b].y; linvel[3 * b + 2] = o->link_lin_vel[b].z;
        angvel[3 * b] = o->link_ang_vel[b].x; angvel[3 * b + 1] = o->link_ang_vel[b].y; angvel[3 * b + 2] = o->link_ang_vel[b].z;
    }
}
}  // extern "C"
