// dm_render_kernel: ray casting of the character's collision shapes from pose rows (the dm_record_pose layout, also a motion-file frame).
// One block per 16 x 16 pixel tile of one view (blockIdx.y); warp 0 computes the view's link frames into shared memory, then every thread
// shades one pixel with one primary ray and, where the light faces the hit, one shadow ray.  tests/render_ref.py restates the arithmetic in
// float64.
#include "dm_render.cuh"

namespace dmk {

namespace {

// ---- shading constants (unscaled metres, linear RGB in [0, 1])
constexpr float kLightX = 0.40824829f, kLightY = 0.81649658f, kLightZ = 0.40824829f;   // towards the light: (1, 2, 1) / sqrt(6)
constexpr float kAmbient = 0.35f, kDiffuse = 0.65f;        // colour = base * (ambient + diffuse * max(n . light, 0) unless shadowed)
constexpr float kCharR = 0.80f, kCharG = 0.45f, kCharB = 0.25f;
constexpr float kMarkR = 0.15f, kMarkG = 0.75f, kMarkB = 0.30f;   // the goal marker (dm_render_poses_marked)
constexpr float kGroundLight = 0.62f, kGroundDark = 0.50f;   // 1 m checker: (floor(x) + floor(z)) even / odd
constexpr float kSkyHorizonR = 0.80f, kSkyHorizonG = 0.87f, kSkyHorizonB = 0.95f;   // at ray y <= 0
constexpr float kSkyZenithR = 0.40f, kSkyZenithG = 0.60f, kSkyZenithB = 0.90f;      // at ray y = 1
constexpr float kTMin = 1e-4f;         // nearest accepted ray parameter
constexpr float kShadowBias = 1e-3f;   // shadow rays start this far along the hit's normal

struct RLink {
    float R[9];     // body frame -> world, row major
    float c[3];     // body frame origin (the collider's centre), world
    float he[3];    // box half extents / capsule radius, half height / sphere radius
    int shape;
};

// nearest hit t > kTMin of the ray o + t d (world) with link L, normal n in world axes; false when none
__device__ __forceinline__ bool hit_link(const RLink& L, V3 o, V3 d, float& t, V3& n) {
    const V3 ow = o - mk3(L.c[0], L.c[1], L.c[2]);
    const V3 lo = mk3(L.R[0] * ow.x + L.R[3] * ow.y + L.R[6] * ow.z, L.R[1] * ow.x + L.R[4] * ow.y + L.R[7] * ow.z, L.R[2] * ow.x + L.R[5] * ow.y + L.R[8] * ow.z);
    const V3 ld = mk3(L.R[0] * d.x + L.R[3] * d.y + L.R[6] * d.z, L.R[1] * d.x + L.R[4] * d.y + L.R[7] * d.z, L.R[2] * d.x + L.R[5] * d.y + L.R[8] * d.z);
    V3 nl;
    if (L.shape == kSBox) {
        float t0 = -INFINITY, t1 = INFINITY;
        int ax = 0;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const float oi = comp(lo, i), di = comp(ld, i), inv = 1.0f / di;
            const float ta = (-L.he[i] - oi) * inv, tb = (L.he[i] - oi) * inv;
            const float tn = fminf(ta, tb), tf = fmaxf(ta, tb);
            if (tn > t0) { t0 = tn; ax = i; }
            t1 = fminf(t1, tf);
        }
        if (!(t0 <= t1 && t0 > kTMin)) return false;
        t = t0;
        nl = (comp(ld, ax) > 0.f ? -1.f : 1.f) * unit3(ax);
    } else {
        // capsule: the side of the cylinder along y within |y| <= half height, and the balls at both ends; a sphere is the ball at the centre
        const float r = L.he[0], h = L.shape == kSCapsule ? L.he[1] : 0.f;
        float best = INFINITY;
        if (L.shape == kSCapsule) {
            const float a = ld.x * ld.x + ld.z * ld.z, b = lo.x * ld.x + lo.z * ld.z, c = lo.x * lo.x + lo.z * lo.z - r * r;
            const float disc = b * b - a * c;
            if (a > 0.f && disc >= 0.f) {
                const float tc = (-b - sqrtf(disc)) / a, y = lo.y + tc * ld.y;
                if (tc > kTMin && fabsf(y) <= h) { best = tc; nl = mk3(lo.x + tc * ld.x, 0.f, lo.z + tc * ld.z); }
            }
        }
#pragma unroll
        for (int s = 0; s < 2; ++s) {
            const V3 oc = lo - mk3(0.f, s ? -h : h, 0.f);
            const float b = dot(oc, ld), c = dot(oc, oc) - r * r, disc = b * b - c;
            if (disc < 0.f) continue;
            const float ts = -b - sqrtf(disc);
            if (ts > kTMin && ts < best) { best = ts; nl = oc + ts * ld; }
        }
        if (!(best < INFINITY)) return false;
        t = best;
        nl = (1.0f / r) * nl;
    }
    n = mk3(L.R[0] * nl.x + L.R[1] * nl.y + L.R[2] * nl.z, L.R[3] * nl.x + L.R[4] * nl.y + L.R[5] * nl.z, L.R[6] * nl.x + L.R[7] * nl.y + L.R[8] * nl.z);
    return true;
}

__device__ __forceinline__ uint8_t to_u8(float c) { return static_cast<uint8_t>(rintf(255.0f * fminf(fmaxf(c, 0.f), 1.f))); }

}  // namespace

// pose: [gridDim.y x pose_dim] rows; rgb [views x height x width x 3] and ids [views x height x width] (-1 sky, -2 ground, k link k), row 0
// at the top; either may be null.
// MARK (dm_render_marked_kernel): an overlay on the plain kernel's output.  marker [gridDim.y x 4] (x, y, z, radius; radius <= 0: none) is a
// sphere hit after the links, shaded like them in a colour of its own (id kRenderMarkerId), and casting shadows like them; the overlay writes
// only the pixels the marker changes -- its own, and the lit ones whose shadow ray only the marker blocks -- so every other pixel keeps the
// plain kernel's bytes
template <bool MARK>
__device__ __forceinline__ void render_body(const DevModel* __restrict__ gm, const float* __restrict__ pose, const float* __restrict__ marker, int width,
                                            int height, RenderCam cam, uint8_t* __restrict__ rgb, int16_t* __restrict__ ids) {
    __shared__ RLink sl[kMaxLinks];
    const DevModel& M = *gm;
    const int nl = M.nl;
    const float* p = pose + static_cast<size_t>(blockIdx.y) * M.pose_dim;
    if constexpr (MARK) {
        if (!(marker[4 * static_cast<size_t>(blockIdx.y) + 3] > 0.f)) return;   // the whole block: one view without a marker
    }
    if (threadIdx.x < 32) {
        // link frames, lane = link (cKinTree::JointWorldTrans as amp_obs_tile walks it): joint frames level by level from att_pt / att_rot and
        // the joint rotations, then each body frame from body_att and child_rot -- the collision pass's link frame, in unscaled metres
        const int lane = threadIdx.x;
        const bool act = lane < nl;
        const DevLink& L = M.link[act ? lane : 0];
        const int plane = L.parent >= 0 ? L.parent : 0, level = act ? L.level : 1000, o = L.pose_off;
        Q4 jq = mkq(0.f, 0.f, 0.f, 1.f);
        if (L.jtype == kJSpherical) jq = qnormalize(mkq(p[o + 1], p[o + 2], p[o + 3], p[o]));
        else if (L.jtype == kJRevolute) { float s, c; sincosf(0.5f * p[o], &s, &c); jq = mkq(0.f, 0.f, s, c); }
        Q4 kq = lane == 0 ? qnormalize(mkq(p[4], p[5], p[6], p[3])) : jq;
        V3 kp = lane == 0 ? mk3(p[0], p[1], p[2]) : mk3(0.f, 0.f, 0.f);
        const V3 att_pt = mk3(L.att_pt[0], L.att_pt[1], L.att_pt[2]);
        const Q4 att_rot = mkq(L.att_rot[0], L.att_rot[1], L.att_rot[2], L.att_rot[3]);
        for (int lv = 1; lv <= M.maxlevel; ++lv) {
            const Q4 pq = mkq(__shfl_sync(0xffffffffu, kq.x, plane), __shfl_sync(0xffffffffu, kq.y, plane), __shfl_sync(0xffffffffu, kq.z, plane),
                              __shfl_sync(0xffffffffu, kq.w, plane));
            const V3 pp = mk3(__shfl_sync(0xffffffffu, kp.x, plane), __shfl_sync(0xffffffffu, kp.y, plane), __shfl_sync(0xffffffffu, kp.z, plane));
            if (level == lv) { kp = pp + qrot(pq, att_pt); kq = qmul(qmul(pq, att_rot), jq); }
        }
        if (act) {
            const Q4 bq = qmul(kq, qconj(mkq(L.child_rot[0], L.child_rot[1], L.child_rot[2], L.child_rot[3])));
            const V3 bp = kp + qrot(kq, mk3(L.body_att[0], L.body_att[1], L.body_att[2]));
            const M3 R = qmat(bq);
            RLink& S = sl[lane];
#pragma unroll
            for (int i = 0; i < 9; ++i) S.R[i] = R.m[i];
            S.c[0] = bp.x; S.c[1] = bp.y; S.c[2] = bp.z;
            const float inv_scale = 1.0f / M.scale;
            S.he[0] = L.he[0] * inv_scale; S.he[1] = L.he[1] * inv_scale; S.he[2] = L.he[2] * inv_scale;
            S.shape = L.shape;
        }
    }
    __syncthreads();
    const int tiles_x = (width + kRenderTile - 1) / kRenderTile;
    const int px = (blockIdx.x % tiles_x) * kRenderTile + threadIdx.x % kRenderTile, py = (blockIdx.x / tiles_x) * kRenderTile + threadIdx.x / kRenderTile;
    if (px >= width || py >= height) return;
    // primary ray through the pixel centre
    const V3 eye = mk3(p[0] + cam.back[0], cam.target_height + cam.back[1], p[2] + cam.back[2]);
    const float sx = (2.0f * (px + 0.5f) / width - 1.0f) * cam.tan_x, sy = (1.0f - 2.0f * (py + 0.5f) / height) * cam.tan_y;
    V3 d = mk3(cam.fwd[0] + sx * cam.right[0] + sy * cam.up[0], cam.fwd[1] + sx * cam.right[1] + sy * cam.up[1], cam.fwd[2] + sx * cam.right[2] + sy * cam.up[2]);
    d = rsqrtf(dot(d, d)) * d;
    float tbest = INFINITY;
    V3 n = mk3(0.f, 1.f, 0.f);
    int id = -1;
    if (d.y < 0.f) {
        const float tg = -eye.y / d.y;
        if (tg > kTMin) { tbest = tg; id = -2; }
    }
    for (int k = 0; k < nl; ++k) {
        float t; V3 nk;
        if (hit_link(sl[k], eye, d, t, nk) && t < tbest) { tbest = t; n = nk; id = k; }
    }
    RLink mk;
    if constexpr (MARK) {
        const float* m = marker + 4 * static_cast<size_t>(blockIdx.y);
#pragma unroll
        for (int i = 0; i < 9; ++i) mk.R[i] = (i % 4 == 0) ? 1.f : 0.f;
        mk.c[0] = m[0]; mk.c[1] = m[1]; mk.c[2] = m[2];
        mk.he[0] = m[3]; mk.he[1] = mk.he[2] = 0.f;
        mk.shape = kSSphere;
        float t; V3 nk;
        if (hit_link(mk, eye, d, t, nk) && t < tbest) { tbest = t; n = nk; id = kRenderMarkerId; }
    }
    const size_t pix = (static_cast<size_t>(blockIdx.y) * height + py) * width + px;
    if (ids && (!MARK || id == kRenderMarkerId)) ids[pix] = static_cast<int16_t>(id);
    if (!rgb) return;
    bool mark_shadow = false;   // MARK: the marker alone blocks the pixel's shadow ray
    float cr, cg, cb;
    if (id == -1) {
        const float s = fmaxf(d.y, 0.f);
        cr = kSkyHorizonR + s * (kSkyZenithR - kSkyHorizonR); cg = kSkyHorizonG + s * (kSkyZenithG - kSkyHorizonG); cb = kSkyHorizonB + s * (kSkyZenithB - kSkyHorizonB);
    } else {
        const V3 P = eye + tbest * d;
        if (id == -2) {
            const float g = ((static_cast<int>(floorf(P.x)) + static_cast<int>(floorf(P.z))) & 1) ? kGroundDark : kGroundLight;
            cr = cg = cb = g;
        } else if (MARK && id == kRenderMarkerId) { cr = kMarkR; cg = kMarkG; cb = kMarkB; }
        else { cr = kCharR; cg = kCharG; cb = kCharB; }
        const V3 light = mk3(kLightX, kLightY, kLightZ);
        const float ndl = dot(n, light);
        float k = kAmbient;
        if (ndl > 0.f) {
            const V3 so = P + kShadowBias * n;
            bool shadow = false;
            for (int j = 0; j < nl && !shadow; ++j) { float t; V3 nj; shadow = hit_link(sl[j], so, light, t, nj); }
            if (MARK && !shadow) { float t; V3 nj; shadow = mark_shadow = hit_link(mk, so, light, t, nj); }
            if (!shadow) k += kDiffuse * ndl;
        }
        cr *= k; cg *= k; cb *= k;
    }
    if (MARK && id != kRenderMarkerId && !mark_shadow) return;
    uint8_t* o = rgb + 3 * pix;
    o[0] = to_u8(cr); o[1] = to_u8(cg); o[2] = to_u8(cb);
}

__global__ void __launch_bounds__(kRenderTile * kRenderTile) dm_render_kernel(const DevModel* __restrict__ gm, const float* __restrict__ pose, int width,
                                                                                int height, RenderCam cam, uint8_t* __restrict__ rgb, int16_t* __restrict__ ids) {
    render_body<false>(gm, pose, nullptr, width, height, cam, rgb, ids);
}
__global__ void __launch_bounds__(kRenderTile * kRenderTile) dm_render_marked_kernel(const DevModel* __restrict__ gm, const float* __restrict__ pose,
                                                                                       const float* __restrict__ marker, int width, int height, RenderCam cam,
                                                                                       uint8_t* __restrict__ rgb, int16_t* __restrict__ ids) {
    render_body<true>(gm, pose, marker, width, height, cam, rgb, ids);
}

}  // namespace dmk
