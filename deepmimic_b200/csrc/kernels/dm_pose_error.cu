// Tracking error of pose rows against reference rows (the dm_record_pose layout), one episode of L frames per column of the [T, n] batch.
// Feature of a pose: every non-root joint's world origin (cKinTree::JointWorldTrans) minus the root's, rotated about y by minus the root's
// heading.  Frame distance d(a, r): the mean over the joints of |f_k(a) - f_k(r)| in metres.  Phase-locked error: the mean of d(a_i, r_i);
// time-warped error: D(L-1, L-1) / 2L of the symmetric DTW recursion D(i, j) = min(D(i-1, j-1) + 2 d_ij, D(i-1, j) + d_ij, D(i, j-1) + d_ij),
// D(0, 0) = 2 d_00.  tests/pose_error_ref.py restates all of it in float64.
//   dm_pose_feature_kernel: one warp per pose row, lane = joint, forward kinematics level by level (dm_render_kernel's walk).
//   dm_pose_dtw_kernel:     one block per episode.  The DP grid runs in strips of kPoseDtwThreads rows, thread t owning row i0 + t, as an
//                           anti-diagonal wavefront: at step s thread t computes column s - t from its left neighbour (its own last value), the
//                           row above (thread t - 1's value of the previous step, through shared memory) and that row's previous value.  The
//                           strip's last row goes to a global boundary row for the next strip.  A thread keeps its row's features in registers;
//                           the reference frames stream through a shared ring of 2 x kPoseDtwThreads columns.  Nothing of the L x L grid is
//                           stored.  The diagonal distances are computed once, summed in row order for the phase-locked error and reused by
//                           the DP, so the diagonal path's value is exactly twice that sum and e_dtw <= e_lock holds in fp32 too.
#include "dm_pose_error.cuh"

namespace dmk {

namespace {

constexpr int kB = kPoseDtwThreads, kRing = 2 * kPoseDtwThreads;

// d(a, r): a in registers, r's component c at r[c * stride]
template <int NJ>
__device__ __forceinline__ float frame_dist(const float (&a)[3 * NJ], const float* r, int stride, int nj, float inv_nj) {
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < NJ; ++k) {
        if (k < nj) {
            const float dx = a[3 * k] - r[(3 * k) * stride], dy = a[3 * k + 1] - r[(3 * k + 1) * stride], dz = a[3 * k + 2] - r[(3 * k + 2) * stride];
            s += sqrtf(dx * dx + dy * dy + dz * dz);
        }
    }
    return s * inv_nj;
}

}  // namespace

__global__ void __launch_bounds__(kPoseFeatureThreads) dm_pose_feature_kernel(const DevModel* __restrict__ gm, const float* __restrict__ a,
                                                                               const float* __restrict__ r, int T, int n, float* __restrict__ feat) {
    const DevModel& M = *gm;
    const int nl = M.nl, F = 3 * (nl - 1);
    const size_t row = static_cast<size_t>(blockIdx.x) * (kPoseFeatureThreads / 32) + threadIdx.x / 32;
    if (row >= static_cast<size_t>(T) * n) return;   // warp-uniform
    const int t = static_cast<int>(row / n), e = static_cast<int>(row % n), lane = threadIdx.x & 31;
    const float* p = (blockIdx.y ? r : a) + row * M.pose_dim;
    const bool act = lane < nl;
    const DevLink& L = M.link[act ? lane : 0];
    const int plane = L.parent >= 0 ? L.parent : 0, level = act ? L.level : 1000, o = L.pose_off;
    Q4 jq = mkq(0.f, 0.f, 0.f, 1.f);
    if (L.jtype == kJSpherical) jq = qnormalize(mkq(p[o + 1], p[o + 2], p[o + 3], p[o]));
    else if (L.jtype == kJRevolute) { float s, c; sincosf(0.5f * p[o], &s, &c); jq = mkq(0.f, 0.f, s, c); }
    const Q4 rq = qnormalize(mkq(p[4], p[5], p[6], p[3]));
    Q4 kq = lane == 0 ? rq : jq;
    const V3 root = mk3(p[0], p[1], p[2]);
    V3 kp = root;
    const V3 att_pt = mk3(L.att_pt[0], L.att_pt[1], L.att_pt[2]);
    const Q4 att_rot = mkq(L.att_rot[0], L.att_rot[1], L.att_rot[2], L.att_rot[3]);
    for (int lv = 1; lv <= M.maxlevel; ++lv) {
        const Q4 pq = mkq(__shfl_sync(0xffffffffu, kq.x, plane), __shfl_sync(0xffffffffu, kq.y, plane), __shfl_sync(0xffffffffu, kq.z, plane),
                          __shfl_sync(0xffffffffu, kq.w, plane));
        const V3 pp = mk3(__shfl_sync(0xffffffffu, kp.x, plane), __shfl_sync(0xffffffffu, kp.y, plane), __shfl_sync(0xffffffffu, kp.z, plane));
        if (level == lv) { kp = pp + qrot(pq, att_pt); kq = qmul(qmul(pq, att_rot), jq); }
    }
    if (lane == 0 || !act) return;
    // heading frame of the root (cKinTree::CalcHeadingRot, as dm_observe_kernel and amp_obs_tile take it): rotation about y by -heading
    const V3 hx = qrot(rq, mk3(1.f, 0.f, 0.f));
    const float heading = atan2f(-hx.z, hx.x);
    float sh, ch; sincosf(-heading, &sh, &ch);
    const V3 d = kp - root;
    float* f = feat + ((static_cast<size_t>(blockIdx.y) * n + e) * T + t) * F + 3 * (lane - 1);
    f[0] = ch * d.x + sh * d.z; f[1] = d.y; f[2] = -sh * d.x + ch * d.z;
}

template <int NJ>
__global__ void __launch_bounds__(kPoseDtwThreads) dm_pose_dtw_kernel(const float* __restrict__ feat, int T, int n, int nj, const int32_t* __restrict__ len,
                                                                      float* bnd, float* __restrict__ lock, float* __restrict__ dtw) {
    extern __shared__ float sr[];          // [3 nj][kRing]: reference frame j's features in column j mod kRing
    __shared__ float sup[2][kB];           // each row's value of the last two steps
    __shared__ float sdiag[kB];            // d(a_i, r_i) of the strip's rows
    const int e = blockIdx.x, t = threadIdx.x;
    const int L = len[e];
    if (L < 1 || L > T) {   // out-of-range length: NaN, nothing read
        if (t == 0) { if (lock) lock[e] = __int_as_float(0x7fc00000); if (dtw) dtw[e] = __int_as_float(0x7fc00000); }
        return;
    }
    const int F = 3 * nj;
    const float inv_nj = 1.0f / nj, inv_len = 1.0f / L, inf = __int_as_float(0x7f800000);
    const float* fa = feat + static_cast<size_t>(e) * T * F;
    const float* fr = feat + (static_cast<size_t>(n) + e) * T * F;
    float* bd = bnd + static_cast<size_t>(e) * T;
    float lock_sum = 0.f;   // thread 0: sum of the diagonal distances in row order
    for (int i0 = 0; i0 < L; i0 += kB) {
        const int i = i0 + t, rows = min(kB, L - i0);
        const bool row_ok = i < L;
        float av[3 * NJ];
#pragma unroll
        for (int c = 0; c < 3 * NJ; ++c) av[c] = (row_ok && c < F) ? fa[static_cast<size_t>(i) * F + c] : 0.f;
        sdiag[t] = row_ok ? frame_dist<NJ>(av, fr + static_cast<size_t>(i) * F, 1, nj, inv_nj) : 0.f;
        float pre = 0.f;   // the next reference column to enter the ring
        if (dtw && t < F) {
            sr[t * kRing] = fr[t];
            if (L > 1) sr[t * kRing + 1] = fr[F + t];
            if (L > 2) pre = fr[2 * F + t];
        }
        __syncthreads();
        if (t == 0)
            for (int k = 0; k < rows; ++k) lock_sum += sdiag[k];
        if (dtw) {
            float left = inf, diag_up = inf;
            float bnext = (t == 0 && i0 > 0) ? bd[0] : inf;
            const int steps = rows + L - 1;
            for (int s = 0; s < steps; ++s) {
                const int j = s - t;
                float up;
                if (t == 0) {
                    up = bnext;
                    if (i0 > 0 && s + 1 < L) bnext = bd[s + 1];
                } else up = sup[(s - 1) & 1][t - 1];
                float D = inf;
                if (row_ok && j >= 0 && j < L) {
                    const float d = j == i ? sdiag[t] : frame_dist<NJ>(av, sr + (j & (kRing - 1)), kRing, nj, inv_nj);
                    const float dg = j == 0 ? inf : diag_up;
                    D = (i == 0 && j == 0) ? 2.f * d : fminf(dg + 2.f * d, fminf(up + d, left + d));
                    left = D;
                    if (t == kB - 1 && i0 + kB < L) bd[j] = D;   // the strip's last row, for the next strip's first
                    if (i == L - 1 && j == L - 1) dtw[e] = (0.5f * D) * inv_len;
                }
                diag_up = up;
                sup[s & 1][t] = D;
                if (t < F && s + 2 < L) {
                    sr[t * kRing + ((s + 2) & (kRing - 1))] = pre;
                    if (s + 3 < L) pre = fr[static_cast<size_t>(s + 3) * F + t];
                }
                __syncthreads();
            }
        }
        __syncthreads();
    }
    if (t == 0 && lock) lock[e] = lock_sum * inv_len;
}
const PoseDtwKernel kPoseDtwKernels[2] = {dm_pose_dtw_kernel<15>, dm_pose_dtw_kernel<31>};

}  // namespace dmk
