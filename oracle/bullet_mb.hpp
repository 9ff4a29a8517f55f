// ORACLE (test infrastructure, not product): single-precision restatement of the part of
// Bullet 2.88 that DeepMimic's hot path runs (SURVEY.md Appendix B):
//   btMultiBody (Featherstone ABA, unit-impulse responses, position integration),
//   btMultiBodyConstraintSolver (PGS over contact / friction / joint-limit rows),
//   btConvexPlaneCollisionAlgorithm + btPersistentManifold (<=4 cached points per link-plane pair).
// Bullet's source is NOT in the reference's repository (un-vendored dependency, pinned tag 2.88, single
// precision: R/README.md:30-40).  Every function below is restated from the published algorithm
// as remembered [B288-mem]; PARITY AGAINST REAL BULLET IS UNPINNED.  Anchors are the reference's
// call sites, cited per function.  Documented simplifications:
//   * link-link (self) collision is not modelled (north_star: capsule/box/sphere vs plane only);
//   * friction rows use the per-row pyramid clamp (the SOLVER_DISABLE_IMPLICIT_CONE_FRICTION path);
//   * warm-start impulses are applied once (v = v_aba + sum_c dV_c * lambda_c).
#pragma once
#include <algorithm>
#include <cassert>
#include <vector>

#include "omath.hpp"

namespace orc {

enum BtJointType { kBtRevolute = 0, kBtSpherical = 2, kBtFixed = 4 };
enum BtShape { kBtBox = 1, kBtCapsule = 2, kBtSphere = 3 };

struct BtManifoldPoint {
    F3 localPointA;       // on the link, link frame
    F3 localPointB;       // on the plane (world == plane frame)
    F3 positionWorldOnA, positionWorldOnB;
    float distance1 = 0;
    float appliedImpulse = 0, appliedImpulseLateral1 = 0, appliedImpulseLateral2 = 0;
    int lifeTime = 0;
};

struct BtManifold {  // btPersistentManifold, MANIFOLD_CACHE_SIZE 4
    BtManifoldPoint pt[4];
    int n = 0;
    float breakingThreshold = 0.02f;
};

struct BtLink {
    float mass = 0;
    F3 inertia;  // diagonal, link frame
    int parent = -1;
    FQ zeroRotParentToThis;
    F3 dVector, eVector;
    int jointType = kBtFixed;
    int dofCount = 0, posVarCount = 0, dofOffset = 0;
    F3 axisTop[3], axisBottom[3];
    float jointPos[4] = {0, 0, 0, 1};
    float jointTorque[3] = {0, 0, 0};
    F3 appliedForce, appliedTorque;
    FQ cachedRotParentToThis;
    F3 cachedRVector;
    // collider
    int shape = kBtSphere;
    F3 halfExtents;  // box: half extents incl. margin; capsule: (radius, halfHeight, -); sphere: (radius,-,-)
    FM3 worldBasis;
    F3 worldPos;
    BtManifold manifold;
    // joint limit (btMultiBodyJointLimitConstraint), revolute only
    bool hasLimit = false;
    float limLow = 0, limHigh = 0;
    // btMultibodyLink::updateCacheMultiDof
    void updateCache() {
        switch (jointType) {
            case kBtRevolute: cachedRotParentToThis = fq_axis_angle(axisTop[0], -jointPos[0]) * zeroRotParentToThis; break;
            case kBtSpherical: cachedRotParentToThis = FQ(jointPos[0], jointPos[1], jointPos[2], -jointPos[3]) * zeroRotParentToThis; break;
            default: cachedRotParentToThis = zeroRotParentToThis; break;
        }
        cachedRVector = dVector + quatRotate(cachedRotParentToThis, eVector);
    }
};

// motion vector [top = angular, bottom = linear]; force vector [lin, ang] kept as the same pair (ang, lin)
struct Sp6 { F3 a, l; };  // a = angular part, l = linear part
inline Sp6 operator+(const Sp6& x, const Sp6& y) { return {x.a + y.a, x.l + y.l}; }
inline Sp6 operator-(const Sp6& x, const Sp6& y) { return {x.a - y.a, x.l - y.l}; }
inline Sp6 operator*(float s, const Sp6& x) { return {s * x.a, s * x.l}; }
inline float spdot(const Sp6& m, const Sp6& f) { return dot(m.a, f.a) + dot(m.l, f.l); }  // motion . force

// btSymmetricSpatialDyad: force = D * motion with  f_lin = TL*w + TR*v,  tau = BL*w + TL^T*v
struct Dyad { FM3 TL = FM3::zero(), TR = FM3::zero(), BL = FM3::zero(); };
inline Sp6 operator*(const Dyad& d, const Sp6& m) { return {d.BL * m.a + transpose(d.TL) * m.l, d.TL * m.a + d.TR * m.l}; }

struct BtContactSolverInfo {  // btContactSolverInfo defaults + the flags the reference sets (sim/World.cpp:67)
    float erp = 0.2f, erp2 = 0.2f, globalCfm = 0.0f, sor = 1.0f, warmstartingFactor = 0.85f;
    float splitImpulsePenetrationThreshold = -0.04f;
    bool splitImpulse = true;
    int numIterations = 10;
    float timeStep = 0;
};

struct SolverRow {  // btMultiBodySolverConstraint
    std::vector<float> jac, deltaV;
    float jacDiagABInv = 0, rhs = 0, cfm = 0, lowerLimit = 0, upperLimit = 0, appliedImpulse = 0, friction = 0;
    int frictionIndex = -1;     // friction rows: index of their normal row
    BtManifoldPoint* pt = nullptr;
};

struct BtMultiBody {
    std::vector<BtLink> links;
    F3 basePos;
    FQ baseQuat;              // world -> base
    std::vector<float> realBuf;  // [omega(3) | vel(3) | joint vel]
    int numDofs = 0;
    float maxCoordinateVelocity = 100.0f, maxAppliedImpulse = 100.0f;
    F3 gravity;
    // ABA cache (valid after computeAccelerationsABA), reused by calcAccelerationDeltas like Bullet does
    std::vector<FM3> rot_from_parent, rot_from_world;
    std::vector<Dyad> spatInertia;
    std::vector<Sp6> h;       // per dof: Ia * axis
    std::vector<float> invD;  // per link dofCount x dofCount block, packed at dofOffset*? (indexed via invDOff)
    std::vector<int> invDOff;
    FM3 cachedTL, cachedTR, cachedLL, cachedLR;  // base articulated inertia blocks
    int n() const { return static_cast<int>(links.size()); }
    // test/debug taps: velocities of the first sub-step of the last stepSimulation call, and the solved impulses
    std::vector<float> dbg_after_aba, dbg_after_pgs, dbg_lambda, dbg_after_aba1, dbg_after_pgs1, dbg_lambda1;
    int dbg_substep = 0;
    // test tap: which branches of the constraint solve each sub-step of the last stepSimulation call took (counts only, no arithmetic)
    struct RowTaps {
        int limits = 0, points = 0;        // joint-limit rows, contact points (solver rows = limits + 3 points)
        int clampAba = 0, clampPgs = 0;    // a generalised velocity hit maxCoordinateVelocity: unconstrained update / applyDeltaVee after PGS
        int limitsAtUpper = 0;             // limit rows whose impulse ended at maxAppliedImpulse
        int frictionSkipped = 0;           // friction rows skipped in the last sweep (their point's normal impulse <= 0)
        int limitsDeep = 0;                // limit rows deeper than the split-impulse threshold (positional term dropped)
    };
    std::vector<RowTaps> dbg_rows;
    // test tap: which branch of the link-plane collision each link took in each sub-step of the last stepSimulation call (no arithmetic)
    enum { kEvNone = 0, kEvAdd = 1, kEvReplace = 2, kEvFull = 3 };
    struct ContactTap {
        int event = kEvNone;   // new point: none, added to a free slot, replaced the nearest cached point, inserted into a full cache
        int slot = -1;         // slot written by the new point
        int deepest = -1;      // full cache: the deepest slot sortCachedPoints kept out of the choice (-1: the new point is the deepest)
        int rmDist = 0;        // refresh: 4-bit masks of the slots (as numbered when the refresh started) removed by distance ...
        int rmDrift = 0;       // ... and by lateral drift of anchor B
        int count = 0;         // points after the refresh
    };
    std::vector<std::vector<ContactTap>> dbg_contacts;

    void finalize() {
        int off = 0;
        invDOff.resize(n());
        int invd = 0;
        for (auto& l : links) { l.dofOffset = off; off += l.dofCount; }
        for (int i = 0; i < n(); ++i) { invDOff[i] = invd; invd += links[i].dofCount * links[i].dofCount; }
        numDofs = off;
        realBuf.assign(6 + numDofs, 0.0f);
        invD.assign(invd, 0.0f);
        h.assign(numDofs, Sp6());
        for (auto& l : links) l.updateCache();
    }
    float* jointVel(int i) { return &realBuf[6 + links[i].dofOffset]; }
    const float* jointVel(int i) const { return &realBuf[6 + links[i].dofOffset]; }

    // btMultiBody::updateCollisionObjectWorldTransforms (call site: sim/SimCharacter.cpp:1214-1217)
    void updateCollisionObjectWorldTransforms() {
        std::vector<FQ> w2l(n() + 1);
        std::vector<F3> org(n() + 1);
        w2l[0] = baseQuat; org[0] = basePos;
        for (int k = 0; k < n(); ++k) {
            int p = links[k].parent;
            w2l[k + 1] = links[k].cachedRotParentToThis * w2l[p + 1];
            org[k + 1] = org[p + 1] + quatRotate(inverse(w2l[k + 1]), links[k].cachedRVector);
            links[k].worldPos = org[k + 1];
            links[k].worldBasis = fm3_from_quat(inverse(w2l[k + 1]));
        }
    }

    // fromParent.transform (btSpatialTransformationMatrix): parent frame -> this frame, motion vectors
    static Sp6 xformM(const FM3& R, const F3& r, const Sp6& in) {
        F3 top = R * in.a;
        return {top, -cross(r, top) + R * in.l};
    }
    // fromParent.transformInverse on a force vector: this frame -> parent frame
    static Sp6 xformInvF(const FM3& R, const F3& r, const Sp6& f) {
        FM3 Rt = transpose(R);
        return {Rt * (f.a + cross(r, f.l)), Rt * f.l};
    }

    // btMultiBody::computeAccelerationsArticulatedBodyAlgorithmMultiDof(dt, ..., isConstraintPass=false)
    // (driven from btMultiBodyDynamicsWorld::solveConstraints; reference call site sim/World.cpp:100)
    void computeAccelerationsABA(float dt) {
        int N = n();
        rot_from_parent.assign(N + 1, FM3()); rot_from_world.assign(N + 1, FM3());
        spatInertia.assign(N + 1, Dyad());
        std::vector<Sp6> spatVel(N + 1), zeroAcc(N + 1), cor(N), spatAcc(N + 1);
        std::vector<float> Y(numDofs, 0.0f), out(6 + numDofs, 0.0f);
        F3 base_omega(realBuf[0], realBuf[1], realBuf[2]), base_vel(realBuf[3], realBuf[4], realBuf[5]);
        rot_from_parent[0] = rot_from_world[0] = fm3_from_quat(baseQuat);
        spatVel[0] = {rot_from_parent[0] * base_omega, rot_from_parent[0] * base_vel};
        zeroAcc[0] = Sp6();  // massless base, no base force (baseMass = 0: sim/SimCharacter.cpp:795-798)
        spatInertia[0] = Dyad();
        for (int i = 0; i < N; ++i) {
            BtLink& L = links[i];
            int p = L.parent;
            rot_from_parent[i + 1] = fm3_from_quat(L.cachedRotParentToThis);
            rot_from_world[i + 1] = rot_from_parent[i + 1] * rot_from_world[p + 1];
            spatVel[i + 1] = xformM(rot_from_parent[i + 1], L.cachedRVector, spatVel[p + 1]);
            Sp6 jv;
            const float* qd = jointVel(i);
            for (int d = 0; d < L.dofCount; ++d) jv = jv + qd[d] * Sp6{L.axisTop[d], L.axisBottom[d]};
            spatVel[i + 1] = spatVel[i + 1] + jv;
            // coriolis: spatVel x jv
            cor[i] = {cross(spatVel[i + 1].a, jv.a), cross(spatVel[i + 1].l, jv.a) + cross(spatVel[i + 1].a, jv.l)};
            // zero-acceleration force: -(external), + gyroscopic terms (m_useGyroTerm = true)
            zeroAcc[i + 1] = {-(rot_from_world[i + 1] * L.appliedTorque), -(rot_from_world[i + 1] * L.appliedForce)};
            F3 Iw(L.inertia.x * spatVel[i + 1].a.x, L.inertia.y * spatVel[i + 1].a.y, L.inertia.z * spatVel[i + 1].a.z);
            zeroAcc[i + 1].a += cross(spatVel[i + 1].a, Iw);
            zeroAcc[i + 1].l += L.mass * cross(spatVel[i + 1].a, spatVel[i + 1].l);
            spatInertia[i + 1].TL = FM3::zero();
            spatInertia[i + 1].TR = FM3::diag(L.mass, L.mass, L.mass);
            spatInertia[i + 1].BL = FM3::diag(L.inertia.x, L.inertia.y, L.inertia.z);
        }
        // second 'downward' loop: articulated inertias and bias forces, leaves -> base
        for (int i = N - 1; i >= 0; --i) {
            BtLink& L = links[i];
            int p = L.parent, nd = L.dofCount;
            float* invDi = nd ? &invD[invDOff[i]] : nullptr;
            float D[9];
            for (int d = 0; d < nd; ++d) {
                Sp6 ax{L.axisTop[d], L.axisBottom[d]};
                h[L.dofOffset + d] = spatInertia[i + 1] * ax;
                Y[L.dofOffset + d] = L.jointTorque[d] - spdot(ax, zeroAcc[i + 1]) - spdot(cor[i], h[L.dofOffset + d]);
            }
            for (int d = 0; d < nd; ++d) for (int d2 = 0; d2 < nd; ++d2) D[d * nd + d2] = spdot(Sp6{L.axisTop[d], L.axisBottom[d]}, h[L.dofOffset + d2]);
            if (nd == 1) invDi[0] = 1.0f / D[0];
            else if (nd == 3) {
                FM3 D3x3; for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) D3x3.m[a][b] = D[a * 3 + b];
                FM3 inv = fm3_inverse(D3x3);
                for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) invDi[a * 3 + b] = inv.m[a][b];
            }
            // Ia -= h invD h^T   (dyad of force vectors), then transform to the parent and add
            Dyad Ia = spatInertia[i + 1];
            for (int d = 0; d < nd; ++d) {
                Sp6 t;  // sum_d2 invD[d][d2] * h[d2]
                for (int d2 = 0; d2 < nd; ++d2) t = t + invDi[d * nd + d2] * h[L.dofOffset + d2];
                const Sp6& hd = h[L.dofOffset + d];
                // symmetric 6x6 [TL TR; BL TL^T] -= hd (x) t   with force layout (lin, ang)
                Ia.TL = Ia.TL - fm3_outer(hd.l, t.a);
                Ia.TR = Ia.TR - fm3_outer(hd.l, t.l);
                Ia.BL = Ia.BL - fm3_outer(hd.a, t.a);
            }
            // shift to parent frame: I_p += X^T Ia X  (btSpatialTransformationMatrix::transformInverse on a dyad)
            {
                const FM3& R = rot_from_parent[i + 1];
                FM3 Rt = transpose(R), rx = fm3_cross(L.cachedRVector);
                // in this frame about the parent's origin: BL' = BL - rx*TL ... (standard parallel-axis for a general dyad)
                FM3 TL = Ia.TL, TR = Ia.TR, BL = Ia.BL;
                // motion from parent-origin frame to COM frame: v_c = v_o + w x r  => v_c = v_o - rx w
                // force back: tau_o = tau_c + r x f_c
                // f = TL w + TR (v_o - rx w)            => TL_o = TL - TR rx ; TR_o = TR
                // tau = BL w + TL^T (v_o - rx w) + rx f => BL_o = BL - TL^T rx + rx (TL - TR rx)
                FM3 TLo = TL - TR * rx;
                FM3 BLo = BL - transpose(TL) * rx + rx * TLo;
                Dyad add;
                add.TL = Rt * TLo * R; add.TR = Rt * TR * R; add.BL = Rt * BLo * R;
                spatInertia[p + 1].TL = spatInertia[p + 1].TL + add.TL;
                spatInertia[p + 1].TR = spatInertia[p + 1].TR + add.TR;
                spatInertia[p + 1].BL = spatInertia[p + 1].BL + add.BL;
            }
            // bias force to the parent
            Sp6 f = zeroAcc[i + 1] + spatInertia[i + 1] * cor[i];
            // NOTE: spatInertia[i+1] keeps the un-reduced articulated inertia like Bullet; Ia (reduced) only goes to the parent.
            for (int d = 0; d < nd; ++d) {
                float s = 0;
                for (int d2 = 0; d2 < nd; ++d2) s += invDi[d * nd + d2] * Y[L.dofOffset + d2];
                f = f + s * h[L.dofOffset + d];
            }
            zeroAcc[p + 1] = zeroAcc[p + 1] + xformInvF(rot_from_parent[i + 1], L.cachedRVector, f);
        }
        // base acceleration: solve Ia_base * a = -zeroAcc[0]
        cachedTL = spatInertia[0].TL; cachedTR = spatInertia[0].TR; cachedLL = spatInertia[0].BL; cachedLR = transpose(spatInertia[0].TL);
        spatAcc[0] = solveImatrix(zeroAcc[0]);
        spatAcc[0] = {-spatAcc[0].a, -spatAcc[0].l};
        for (int i = 0; i < N; ++i) {
            BtLink& L = links[i];
            int p = L.parent, nd = L.dofCount;
            spatAcc[i + 1] = xformM(rot_from_parent[i + 1], L.cachedRVector, spatAcc[p + 1]);
            float ymh[3];
            for (int d = 0; d < nd; ++d) ymh[d] = Y[L.dofOffset + d] - spdot(spatAcc[i + 1], h[L.dofOffset + d]);
            const float* invDi = nd ? &invD[invDOff[i]] : nullptr;
            spatAcc[i + 1] = spatAcc[i + 1] + cor[i];
            for (int d = 0; d < nd; ++d) {
                float qdd = 0;
                for (int d2 = 0; d2 < nd; ++d2) qdd += invDi[d * nd + d2] * ymh[d2];
                out[6 + L.dofOffset + d] = qdd;
                spatAcc[i + 1] = spatAcc[i + 1] + qdd * Sp6{L.axisTop[d], L.axisBottom[d]};
            }
        }
        FM3 R0t = transpose(rot_from_parent[0]);
        F3 wd = R0t * spatAcc[0].a;
        F3 vd = R0t * (spatAcc[0].l + cross(spatVel[0].a, spatVel[0].l));
        out[0] = wd.x; out[1] = wd.y; out[2] = wd.z; out[3] = vd.x; out[4] = vd.y; out[5] = vd.z;
        const bool clamped = applyDeltaVee(out.data(), dt);
        if (!dbg_rows.empty()) dbg_rows.back().clampAba = clamped ? 1 : 0;
    }

    // btMultiBody::solveImatrix: x = Ia_base^-1 * rhs (block inverse of the 6x6 base articulated inertia)
    Sp6 solveImatrix(const Sp6& rhs) const {
        // [f_lin; tau] = [TL TR; LL LR] [w; v]   -> solve for (w, v) given rhs = (tau = rhs.a, f_lin = rhs.l)
        FM3 Binv = fm3_inverse(cachedTR);
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) Binv.m[i][j] *= -1.0f;
        FM3 tmp = cachedLR * Binv;
        FM3 invIupper_right = fm3_inverse(tmp * cachedTL + cachedLL);
        tmp = invIupper_right * cachedLR;
        FM3 invI_upper_left = tmp * Binv;
        FM3 invI_lower_right = transpose(invI_upper_left);
        tmp = cachedTL * invI_upper_left;
        tmp.m[0][0] -= 1.0f; tmp.m[1][1] -= 1.0f; tmp.m[2][2] -= 1.0f;
        FM3 invI_lower_left = Binv * tmp;
        F3 vtop = invI_upper_left * rhs.l + invIupper_right * rhs.a;
        F3 vbot = invI_lower_left * rhs.l + invI_lower_right * rhs.a;
        return {vtop, vbot};
    }

    // btMultiBody::applyDeltaVeeMultiDof; returns whether a coordinate was clamped
    bool applyDeltaVee(const float* dv, float mult) {
        bool clamped = false;
        for (int d = 0; d < 6 + numDofs; ++d) {
            realBuf[d] += dv[d] * mult;
            clamped |= std::fabs(realBuf[d]) > maxCoordinateVelocity;
            realBuf[d] = std::min(std::max(realBuf[d], -maxCoordinateVelocity), maxCoordinateVelocity);
        }
        return clamped;
    }

    // btMultiBody::calcAccelerationDeltasMultiDof: out = M^-1 * force (generalised), reusing the ABA cache
    void calcAccelerationDeltas(const float* force, float* out) const {
        int N = n();
        std::vector<Sp6> zeroAcc(N + 1), spatAcc(N + 1);
        std::vector<float> Y(numDofs, 0.0f);
        zeroAcc[0] = {-(rot_from_parent[0] * F3(force[0], force[1], force[2])), -(rot_from_parent[0] * F3(force[3], force[4], force[5]))};
        for (int i = N - 1; i >= 0; --i) {
            const BtLink& L = links[i];
            int p = L.parent, nd = L.dofCount;
            const float* invDi = nd ? &invD[invDOff[i]] : nullptr;
            for (int d = 0; d < nd; ++d) Y[L.dofOffset + d] = force[6 + L.dofOffset + d] - spdot(Sp6{L.axisTop[d], L.axisBottom[d]}, zeroAcc[i + 1]);
            Sp6 f = zeroAcc[i + 1];
            for (int d = 0; d < nd; ++d) {
                float s = 0;
                for (int d2 = 0; d2 < nd; ++d2) s += invDi[d * nd + d2] * Y[L.dofOffset + d2];
                f = f + s * h[L.dofOffset + d];
            }
            zeroAcc[p + 1] = zeroAcc[p + 1] + xformInvF(rot_from_parent[i + 1], L.cachedRVector, f);
        }
        Sp6 r = solveImatrix(zeroAcc[0]);
        spatAcc[0] = {-r.a, -r.l};
        for (int i = 0; i < N; ++i) {
            const BtLink& L = links[i];
            int p = L.parent, nd = L.dofCount;
            spatAcc[i + 1] = xformM(rot_from_parent[i + 1], L.cachedRVector, spatAcc[p + 1]);
            float ymh[3];
            for (int d = 0; d < nd; ++d) ymh[d] = Y[L.dofOffset + d] - spdot(spatAcc[i + 1], h[L.dofOffset + d]);
            const float* invDi = nd ? &invD[invDOff[i]] : nullptr;
            for (int d = 0; d < nd; ++d) {
                float qdd = 0;
                for (int d2 = 0; d2 < nd; ++d2) qdd += invDi[d * nd + d2] * ymh[d2];
                out[6 + L.dofOffset + d] = qdd;
                spatAcc[i + 1] = spatAcc[i + 1] + qdd * Sp6{L.axisTop[d], L.axisBottom[d]};
            }
        }
        FM3 R0t = transpose(rot_from_parent[0]);
        F3 wd = R0t * spatAcc[0].a, vd = R0t * spatAcc[0].l;
        out[0] = wd.x; out[1] = wd.y; out[2] = wd.z; out[3] = vd.x; out[4] = vd.y; out[5] = vd.z;
    }

    // btMultiBody::fillConstraintJacobianMultiDof(link, contact_point, normal_ang = 0, normal_lin)
    void fillContactJacobian(int link, const F3& contact_point, const F3& normal, float* jac) const {
        int N = n();
        std::vector<F3> pmc(N + 1), nl(N + 1);
        std::vector<float> results(numDofs, 0.0f);
        F3 p_minus_com_world = contact_point - basePos;
        FM3 rw0 = fm3_from_quat(baseQuat);
        F3 oc = cross(p_minus_com_world, normal);
        jac[0] = oc.x; jac[1] = oc.y; jac[2] = oc.z; jac[3] = normal.x; jac[4] = normal.y; jac[5] = normal.z;
        pmc[0] = rw0 * p_minus_com_world; nl[0] = rw0 * normal;
        for (int i = 6; i < 6 + numDofs; ++i) jac[i] = 0;
        for (int i = 0; i < N; ++i) {
            const BtLink& L = links[i];
            int p = L.parent;
            FM3 mtx = fm3_from_quat(L.cachedRotParentToThis);
            nl[i + 1] = mtx * nl[p + 1];
            pmc[i + 1] = mtx * pmc[p + 1] - L.cachedRVector;
            for (int d = 0; d < L.dofCount; ++d) results[L.dofOffset + d] = dot(nl[i + 1], cross(L.axisTop[d], pmc[i + 1]) + L.axisBottom[d]);
        }
        while (link != -1) {
            for (int d = 0; d < links[link].dofCount; ++d) jac[6 + links[link].dofOffset + d] = results[links[link].dofOffset + d];
            link = links[link].parent;
        }
    }

    // btMultiBody::stepPositionsMultiDof(dt)
    void stepPositions(float dt) {
        basePos.x += dt * realBuf[3]; basePos.y += dt * realBuf[4]; basePos.z += dt * realBuf[5];
        auto quatUpdate = [](const F3& omega, FQ& quat, bool baseBody, float dt) {
            F3 angvel = baseBody ? omega : quatRotate(quat, omega);
            float fAngle = length(angvel);
            const float ANGULAR_MOTION_THRESHOLD = 0.5f * 1.57079632679489661923f;
            if (fAngle * dt > ANGULAR_MOTION_THRESHOLD) fAngle = 0.5f * 1.57079632679489661923f / dt;
            F3 axis;
            if (fAngle < 0.001f) axis = angvel * (0.5f * dt - (dt * dt * dt) * 0.020833333333f * fAngle * fAngle);
            else axis = angvel * (std::sin(0.5f * fAngle * dt) / fAngle);
            if (!baseBody) quat = FQ(axis.x, axis.y, axis.z, std::cos(fAngle * dt * 0.5f)) * quat;
            else quat = quat * FQ(-axis.x, -axis.y, -axis.z, std::cos(fAngle * dt * 0.5f));
            quat = normalized(quat);
        };
        quatUpdate(F3(realBuf[0], realBuf[1], realBuf[2]), baseQuat, true, dt);
        for (int i = 0; i < n(); ++i) {
            BtLink& L = links[i];
            const float* qd = jointVel(i);
            if (L.jointType == kBtRevolute) L.jointPos[0] += dt * qd[0];
            else if (L.jointType == kBtSpherical) {
                FQ ori(L.jointPos[0], L.jointPos[1], L.jointPos[2], L.jointPos[3]);
                quatUpdate(F3(qd[0], qd[1], qd[2]), ori, false, dt);
                L.jointPos[0] = ori.x; L.jointPos[1] = ori.y; L.jointPos[2] = ori.z; L.jointPos[3] = ori.w;
            }
            L.updateCache();
        }
    }

    // ------------------------------------------------------------------ collision: link convex vs y=0 plane
    // convex->localGetSupportingVertex(dir) [btBoxShape / btCapsuleShape / btSphereShape]
    static F3 supportVertex(const BtLink& L, const F3& vec) {
        if (L.shape == kBtBox) {
            const F3& he = L.halfExtents;
            return F3(vec.x >= 0 ? he.x : -he.x, vec.y >= 0 ? he.y : -he.y, vec.z >= 0 ? he.z : -he.z);
        }
        F3 sup(0, 0, 0);
        float radius = L.halfExtents.x;
        if (L.shape == kBtCapsule) {
            F3 v = vec;
            float lenSqr = dot(v, v);
            if (lenSqr < 0.0001f) v = F3(1, 0, 0); else v = v * (1.0f / std::sqrt(lenSqr));
            float hh = L.halfExtents.y;
            float maxDot = -1e18f;
            F3 p1(0, hh, 0), p2(0, -hh, 0);
            float d1 = dot(v, p1); if (d1 > maxDot) { maxDot = d1; sup = p1; }
            float d2 = dot(v, p2); if (d2 > maxDot) { maxDot = d2; sup = p2; }
        }
        // btConvexInternalShape::localGetSupportingVertex: + margin * normalized(vec); margin == radius here
        F3 vn = vec;
        if (dot(vn, vn) < 1.1920929e-7f * 1.1920929e-7f) vn = F3(-1, -1, -1);
        vn = vn * (1.0f / length(vn));
        return sup + radius * vn;
    }
    // btPersistentManifold::sortCachedPoints (KEEP_DEEPEST_POINT, gContactCalcArea3Points = true)
    static int sortCachedPoints(const BtManifold& m, const BtManifoldPoint& pt, int* deepest = nullptr) {
        int maxPenetrationIndex = -1;
        float maxPenetration = pt.distance1;
        for (int i = 0; i < 4; ++i) if (m.pt[i].distance1 < maxPenetration) { maxPenetrationIndex = i; maxPenetration = m.pt[i].distance1; }
        float res[4] = {0, 0, 0, 0};
        auto area = [&](const F3& a, const F3& b) { F3 c = cross(a, b); return dot(c, c); };
        if (maxPenetrationIndex != 0) res[0] = area(pt.localPointA - m.pt[1].localPointA, m.pt[3].localPointA - m.pt[2].localPointA);
        if (maxPenetrationIndex != 1) res[1] = area(pt.localPointA - m.pt[0].localPointA, m.pt[3].localPointA - m.pt[2].localPointA);
        if (maxPenetrationIndex != 2) res[2] = area(pt.localPointA - m.pt[0].localPointA, m.pt[3].localPointA - m.pt[1].localPointA);
        if (maxPenetrationIndex != 3) res[3] = area(pt.localPointA - m.pt[0].localPointA, m.pt[2].localPointA - m.pt[1].localPointA);
        int best = -1; float bv = -1e18f;
        for (int i = 0; i < 4; ++i) if (std::fabs(res[i]) > bv) { bv = std::fabs(res[i]); best = i; }
        if (deepest) *deepest = maxPenetrationIndex;
        return best;
    }
    // btConvexPlaneCollisionAlgorithm::processCollision (one new point per frame, numPerturbationIterations gated off)
    // + btManifoldResult::addContactPoint + btPersistentManifold::refreshContactPoints
    void collideLinkPlane(int i) {
        BtLink& L = links[i];
        BtManifold& m = L.manifold;
        ContactTap tap;
        const F3 n(0, 1, 0);
        F3 dirLocal = transpose(L.worldBasis) * (-n);
        F3 vtx = supportVertex(L, dirLocal);
        F3 vtxInPlane = L.worldBasis * vtx + L.worldPos;
        float distance = dot(n, vtxInPlane);  // plane constant 0
        F3 projected = vtxInPlane - distance * n;
        if (distance < m.breakingThreshold) {
            // addContactPoint(normalOnB = n, pointInWorld = projected, depth = distance)
            if (!(distance > m.breakingThreshold)) {
                F3 pointA = projected + distance * n;
                BtManifoldPoint np;
                np.localPointA = transpose(L.worldBasis) * (pointA - L.worldPos);
                np.localPointB = projected;
                np.positionWorldOnA = pointA; np.positionWorldOnB = projected; np.distance1 = distance;
                // getCacheEntry
                float shortest = m.breakingThreshold * m.breakingThreshold;
                int nearest = -1;
                for (int k = 0; k < m.n; ++k) {
                    F3 d = m.pt[k].localPointA - np.localPointA;
                    float dd = dot(d, d);
                    if (dd < shortest) { shortest = dd; nearest = k; }
                }
                if (nearest >= 0) {  // replaceContactPoint keeps impulses and lifetime
                    np.appliedImpulse = m.pt[nearest].appliedImpulse;
                    np.appliedImpulseLateral1 = m.pt[nearest].appliedImpulseLateral1;
                    np.appliedImpulseLateral2 = m.pt[nearest].appliedImpulseLateral2;
                    np.lifeTime = m.pt[nearest].lifeTime;
                    m.pt[nearest] = np;
                    tap.event = kEvReplace; tap.slot = nearest;
                } else {  // addManifoldPoint
                    int idx = m.n;
                    tap.event = kEvAdd;
                    if (idx == 4) { idx = sortCachedPoints(m, np, &tap.deepest); tap.event = kEvFull; } else m.n++;
                    if (idx < 0) idx = 0;
                    m.pt[idx] = np;
                    tap.slot = idx;
                }
            }
        }
        // refreshContactPoints
        for (int k = m.n - 1; k >= 0; --k) {
            BtManifoldPoint& p = m.pt[k];
            p.positionWorldOnA = L.worldBasis * p.localPointA + L.worldPos;
            p.positionWorldOnB = p.localPointB;
            p.distance1 = dot(p.positionWorldOnA - p.positionWorldOnB, n);
            p.lifeTime++;
        }
        for (int k = m.n - 1; k >= 0; --k) {
            BtManifoldPoint& p = m.pt[k];
            bool remove = false;
            if (!(p.distance1 <= m.breakingThreshold)) remove = true;
            else {
                F3 projectedPoint = p.positionWorldOnA - p.distance1 * n;
                F3 diff = p.positionWorldOnB - projectedPoint;
                if (dot(diff, diff) > m.breakingThreshold * m.breakingThreshold) remove = true;
            }
            if (remove) {
                (p.distance1 <= m.breakingThreshold ? tap.rmDrift : tap.rmDist) |= 1 << k;
                int last = m.n - 1; if (k != last) m.pt[k] = m.pt[last]; m.n--;
            }
        }
        tap.count = m.n;
        if (!dbg_contacts.empty()) dbg_contacts.back()[i] = tap;
    }

    // ------------------------------------------------------------------ constraint solve
    // btMultiBodyConstraintSolver::solveGroup (setup / 10 PGS iterations / finish) for one multibody vs the static plane
    void solveConstraints(const BtContactSolverInfo& info, float friction) {
        const int nd = 6 + numDofs;
        std::vector<SolverRow> normals, frictions, limits;
        std::vector<float> deltaVelocities(nd, 0.0f);
        const F3 nrm(0, 1, 0);
        const F3 t1(-1, 0, 0), t2(0, 0, 1);  // btPlaneSpace1((0,1,0))
        auto relVel = [&](const std::vector<float>& jac) { float s = 0; for (int k = 0; k < nd; ++k) s += realBuf[k] * jac[k]; return s; };
        auto makeRow = [&](int link, const F3& pos, const F3& dir) {
            SolverRow r;
            r.jac.assign(nd, 0.0f); r.deltaV.assign(nd, 0.0f);
            fillContactJacobian(link, pos, dir, r.jac.data());
            calcAccelerationDeltas(r.jac.data(), r.deltaV.data());
            float denom = 0; for (int k = 0; k < nd; ++k) denom += r.jac[k] * r.deltaV[k];
            float d = denom + info.globalCfm;
            r.jacDiagABInv = (d > 1.1920929e-7f) ? info.sor / d : 0.0f;
            return r;
        };
        // convertContacts: btMultiBodyConstraintSolver::convertMultiBodyContact / setupMultiBodyContactConstraint
        for (int i = 0; i < n(); ++i) {
            BtManifold& m = links[i].manifold;
            for (int k = 0; k < m.n; ++k) {
                BtManifoldPoint& cp = m.pt[k];
                SolverRow r = makeRow(i, cp.positionWorldOnA, nrm);
                r.pt = &cp;
                float rel_vel = relVel(r.jac);
                float penetration = cp.distance1;  // + linearSlop (0)
                float positionalError = 0.0f, velocityError = 0.0f - rel_vel;  // restitution 0
                float erp = info.erp2;
                if (!info.splitImpulse || penetration > info.splitImpulsePenetrationThreshold) erp = info.erp;
                if (penetration > 0) { positionalError = 0; velocityError -= penetration / info.timeStep; }
                else positionalError = -penetration * erp / info.timeStep;
                r.rhs = positionalError * r.jacDiagABInv + velocityError * r.jacDiagABInv;
                r.cfm = info.globalCfm * r.jacDiagABInv;
                r.lowerLimit = 0; r.upperLimit = 1e10f;
                r.friction = friction;
                r.appliedImpulse = cp.appliedImpulse * info.warmstartingFactor;  // SOLVER_USE_WARMSTARTING
                if (r.appliedImpulse != 0.0f) for (int q = 0; q < nd; ++q) deltaVelocities[q] += r.deltaV[q] * r.appliedImpulse;
                int normalIdx = static_cast<int>(normals.size());
                normals.push_back(r);
                for (int f = 0; f < 2; ++f) {  // SOLVER_USE_2_FRICTION_DIRECTIONS
                    SolverRow fr = makeRow(i, cp.positionWorldOnA, f == 0 ? t1 : t2);
                    fr.pt = &cp;
                    float rv = relVel(fr.jac);
                    fr.rhs = (0.0f - rv) * fr.jacDiagABInv;
                    fr.cfm = info.globalCfm * fr.jacDiagABInv;
                    fr.friction = friction; fr.lowerLimit = -friction; fr.upperLimit = friction;
                    fr.appliedImpulse = 0;  // friction rows are not warm started in the multibody solver
                    fr.frictionIndex = normalIdx;
                    frictions.push_back(fr);
                }
            }
        }
        // btMultiBodyJointLimitConstraint::createConstraintRows (constraints built at sim/SimCharacter.cpp:948-973)
        for (int i = 0; i < n(); ++i) {
            BtLink& L = links[i];
            if (!L.hasLimit) continue;
            float pos[2] = {L.jointPos[0] - L.limLow, L.limHigh - L.jointPos[0]};
            for (int row = 0; row < 2; ++row) {
                float penetration = pos[row];
                if (penetration > 0) continue;
                float direction = row ? -1.0f : 1.0f;
                SolverRow r;
                r.jac.assign(nd, 0.0f); r.deltaV.assign(nd, 0.0f);
                r.jac[6 + L.dofOffset] = direction;
                calcAccelerationDeltas(r.jac.data(), r.deltaV.data());
                float denom = 0; for (int k = 0; k < nd; ++k) denom += r.jac[k] * r.deltaV[k];
                float d = denom + info.globalCfm;
                r.jacDiagABInv = (d > 1.1920929e-7f) ? info.sor / d : 0.0f;
                float rel_vel = relVel(r.jac);
                float positionalError = 0.0f, velocityError = -rel_vel;
                float erp = info.erp2;
                bool combine = (!info.splitImpulse || penetration > info.splitImpulsePenetrationThreshold);
                if (combine) erp = info.erp;
                if (penetration > 0) { positionalError = 0; velocityError = -penetration / info.timeStep; }
                else positionalError = -penetration * erp / info.timeStep;
                float penetrationImpulse = positionalError * r.jacDiagABInv, velocityImpulse = velocityError * r.jacDiagABInv;
                r.rhs = combine ? penetrationImpulse + velocityImpulse : velocityImpulse;  // m_rhsPenetration is never consumed for multibodies
                r.cfm = 0; r.lowerLimit = 0; r.upperLimit = maxAppliedImpulse; r.appliedImpulse = 0;
                limits.push_back(r);
                if (!combine && !dbg_rows.empty()) dbg_rows.back().limitsDeep++;
            }
        }
        // resolveSingleConstraintRowGeneric
        auto resolve = [&](SolverRow& c) {
            float deltaImpulse = c.rhs - c.appliedImpulse * c.cfm;
            float dvdotn = 0; for (int k = 0; k < nd; ++k) dvdotn += c.jac[k] * deltaVelocities[k];
            deltaImpulse -= dvdotn * c.jacDiagABInv;
            float sum = c.appliedImpulse + deltaImpulse;
            if (sum < c.lowerLimit) { deltaImpulse = c.lowerLimit - c.appliedImpulse; c.appliedImpulse = c.lowerLimit; }
            else if (sum > c.upperLimit) { deltaImpulse = c.upperLimit - c.appliedImpulse; c.appliedImpulse = c.upperLimit; }
            else c.appliedImpulse = sum;
            for (int k = 0; k < nd; ++k) deltaVelocities[k] += c.deltaV[k] * deltaImpulse;
        };
        // btMultiBodyConstraintSolver::solveSingleIteration x numIterations (SOLVER_FRICTION_SEPARATE ordering)
        for (int it = 0; it < info.numIterations; ++it) {
            int nl = static_cast<int>(limits.size());
            for (int j = 0; j < nl; ++j) resolve(limits[(it & 1) ? j : nl - 1 - j]);
            for (auto& c : normals) resolve(c);
            int skipped = 0;
            for (auto& c : frictions) {
                float totalImpulse = normals[c.frictionIndex].appliedImpulse;
                if (totalImpulse > 0) { c.lowerLimit = -(c.friction * totalImpulse); c.upperLimit = c.friction * totalImpulse; resolve(c); }
                else skipped++;
            }
            if (it == info.numIterations - 1 && !dbg_rows.empty()) dbg_rows.back().frictionSkipped = skipped;
        }
        // finish: velocities += accumulated delta (clamped like applyDeltaVeeMultiDof), impulses written back to the manifold
        const bool clamped = applyDeltaVee(deltaVelocities.data(), 1.0f);
        if (!dbg_rows.empty()) {
            RowTaps& t = dbg_rows.back();
            t.limits = static_cast<int>(limits.size()); t.points = static_cast<int>(normals.size()); t.clampPgs = clamped ? 1 : 0;
            for (auto& c : limits) t.limitsAtUpper += (c.appliedImpulse == c.upperLimit) ? 1 : 0;
        }
        if (dbg_substep == 1) { dbg_lambda1.clear(); for (auto& c : normals) dbg_lambda1.push_back(c.appliedImpulse); for (auto& c : frictions) dbg_lambda1.push_back(c.appliedImpulse); for (auto& c : limits) dbg_lambda1.push_back(c.appliedImpulse); }
        if (dbg_substep == 0) { dbg_lambda.clear(); for (auto& c : normals) dbg_lambda.push_back(c.appliedImpulse); for (auto& c : frictions) dbg_lambda.push_back(c.appliedImpulse); for (auto& c : limits) dbg_lambda.push_back(c.appliedImpulse); }
        for (size_t k = 0; k < normals.size(); ++k) {
            normals[k].pt->appliedImpulse = normals[k].appliedImpulse;
            normals[k].pt->appliedImpulseLateral1 = frictions[2 * k].appliedImpulse;
            normals[k].pt->appliedImpulseLateral2 = frictions[2 * k + 1].appliedImpulse;
        }
    }

    // btDiscreteDynamicsWorld::internalSingleStepSimulation for one multibody (reference call site sim/World.cpp:93-104)
    void internalSingleStep(float h, const BtContactSolverInfo& base_info, float friction) {
        dbg_contacts.emplace_back(n());
        for (int i = 0; i < n(); ++i) collideLinkPlane(i);          // performDiscreteCollisionDetection
        dbg_rows.emplace_back();
        computeAccelerationsABA(h);                                  // solveConstraints: ABA, v += a h
        if (dbg_substep == 0) dbg_after_aba = realBuf; else if (dbg_substep == 1) dbg_after_aba1 = realBuf;
        BtContactSolverInfo info = base_info; info.timeStep = h;
        solveConstraints(info, friction);                            // PGS
        if (dbg_substep == 0) dbg_after_pgs = realBuf; else if (dbg_substep == 1) dbg_after_pgs1 = realBuf;
        dbg_substep++;
        stepPositions(h);                                            // integrateTransforms
        updateCollisionObjectWorldTransforms();
    }
    // btDiscreteDynamicsWorld::stepSimulation(timeStep, maxSubSteps, fixedTimeStep) with applyGravity / clearForces
    void stepSimulation(float timeStep, int maxSubSteps, float fixedTimeStep, const BtContactSolverInfo& info, float friction) {
        int numSub = static_cast<int>(timeStep / fixedTimeStep);  // m_localTime starts at 0 and returns to 0 every call
        numSub = std::min(numSub, maxSubSteps);
        for (auto& L : links) L.appliedForce += L.mass * gravity;   // applyGravity (btMultiBodyDynamicsWorld)
        dbg_substep = 0;
        dbg_rows.clear();
        dbg_contacts.clear();
        for (int s = 0; s < numSub; ++s) internalSingleStep(fixedTimeStep, info, friction);
        for (auto& L : links) { L.appliedForce = F3(); L.appliedTorque = F3(); L.jointTorque[0] = L.jointTorque[1] = L.jointTorque[2] = 0; }  // clearForces
    }
    void clearContacts() { for (auto& L : links) L.manifold.n = 0; }
};

}  // namespace orc
