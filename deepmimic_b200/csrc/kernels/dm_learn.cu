// The PPO learner's minibatch step on the device (R/learning/ppo_agent.py: PPOAgent._update_actor / _update_critic, solvers/mpi_solver.py) for
// the plain 2-layer networks, around the wgmma GEMMs of kernels/dm_mlp.cu (forward: the inference kernels; backward: dm_mlp_grad_x_kernel,
// dm_mlp_grad_w_kernel):
//   * operand preparation that gathers the minibatch's rows from the [samples x in_dim] window by a device index array,
//   * the transposition of the saved forward activations into the dW GEMM's A operand (M = features + a ones feature whose dW row is db),
//   * one loss head per network: per row the clipped-surrogate + bound-loss gradient (actor) or the value-loss gradient (critic) w.r.t. the
//     normalised output, written as hi + lo fp16 tiles for the dX GEMM (A) and the dW GEMM (B).  dY is the gradient of the SUM over
//     rows (per-row actor gradients reach ~1e2; scaled by 1/B they would sink toward fp16's subnormals); 1/B is applied in fp32 by the
//     optimiser.  Rows past the minibatch carry dY = 0 (the forward writes relu(bias) there).  The losses and the clip count are reduced per
//     CTA in a fixed tree and summed in a fixed order by one thread (no float atomics: the step is bit-reproducible),
//   * one elementwise pass per layer: the split-K dW partials summed in a fixed order, weight decay on weights (not biases), the momentum step
//     acc = m acc + g, w -= lr acc (TF MomentumOptimizer) on the fp32 torch parameters, and the re-tiling of the new weights into the forward
//     hi + lo tiles and the transposed tiles of the next dX GEMM.  Without an optimiser step the same pass re-tiles fp32 device weights into a
//     dm_mlp handle (dm_mlp_set_weights_device).
// The AMP discriminator's step (dm_learn_disc_step) reuses the preparation, transposition and backward GEMMs and adds its least-squares head
// (which also seeds dd/dd = 1 on the expert rows for the gradient penalty), the per-row ||dd/dx||^2 partials, its statistics and a layer pass
// that adds the penalty's weight gradients and the logit regulariser.  The gated networks' step (dm_learn_gated_step) adds a preparation that
// also writes the goal's tile and reuses the rest; its gated backward epilogue is in kernels/dm_mlp.cu (GRAD_XG).
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cstdint>

#include "dm_mlp.cuh"

namespace dmk {

constexpr int kLearnRows = 128;        // rows per CTA of the preparation, transposition and head kernels (one m tile)

// minibatch rows gathered from the window -> normalised, clipped fp16 operand tiles (dm_mlp_prep_kernel with a row index)
__global__ void __launch_bounds__(kLearnRows) dm_learn_prep_kernel(LearnPrepParams P) {
    const int m0 = blockIdx.x * kLearnRows, c = blockIdx.y;
    __half* tile = P.tiles + (static_cast<size_t>(blockIdx.x) * P.NC + c) * kMlpATile;
#pragma unroll
    for (int i = 0; i < (kLearnRows * 8) / kLearnRows; ++i) {
        const int u = threadIdx.x + i * kLearnRows, row = u >> 3, k8 = u & 7;
        const int grow = m0 + row, k = c * 64 + k8 * 8;
        const float* src = grow < P.M ? P.x + static_cast<size_t>(P.idx[grow]) * P.in_dim : nullptr;
        __align__(16) __half h[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            float x = 0.f;
            if (src && k + e < P.in_dim) x = fminf(fmaxf((src[k + e] - P.mean[k + e]) * P.istd[k + e], -P.clip), P.clip);
            h[e] = __float2half_rn(x);
        }
        *reinterpret_cast<uint4*>(tile + ((k8 * (kLearnRows / 8) + (row >> 3)) * 64 + (row & 7) * 8)) = *reinterpret_cast<const uint4*>(h);
    }
}

// dm_learn_prep_kernel for the gated networks: the trunk tiles hold [state | goal] and the extra chunk blockIdx.y == NC writes the normalised
// goal's own tile, as dm_mlp_gated_prep_kernel does.  (A kernel of its own: sharing the body changes dm_learn_prep_kernel's code.)
// grid = (m tiles, NC + 1)
__global__ void __launch_bounds__(kLearnRows) dm_learn_gated_prep_kernel(LearnPrepParams P, LearnGoalParams Q) {
    const int m0 = blockIdx.x * kLearnRows;
    const bool gate = static_cast<int>(blockIdx.y) == P.NC;
    const int c = gate ? 0 : blockIdx.y;
    __half* tile = gate ? Q.g_tiles + static_cast<size_t>(blockIdx.x) * kMlpATile : P.tiles + (static_cast<size_t>(blockIdx.x) * P.NC + c) * kMlpATile;
#pragma unroll
    for (int i = 0; i < (kLearnRows * 8) / kLearnRows; ++i) {
        const int u = threadIdx.x + i * kLearnRows, row = u >> 3, k8 = u & 7;
        const int grow = m0 + row, k = c * 64 + k8 * 8;
        const int64_t s = grow < P.M ? P.idx[grow] : -1;
        __align__(16) __half h[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            float x = 0.f;
            if (s >= 0 && !gate && k + e < P.in_dim) {
                x = fminf(fmaxf((P.x[s * P.in_dim + k + e] - P.mean[k + e]) * P.istd[k + e], -P.clip), P.clip);
            } else if (s >= 0) {
                const int j = gate ? k + e : k + e - P.in_dim;
                if (j < Q.goal_dim) x = fminf(fmaxf((Q.goal[s * Q.goal_dim + j] - Q.g_mean[j]) * Q.g_istd[j], -Q.g_clip), Q.g_clip);
            }
            h[e] = __float2half_rn(x);
        }
        *reinterpret_cast<uint4*>(tile + ((k8 * (kLearnRows / 8) + (row >> 3)) * 64 + (row & 7) * 8)) = *reinterpret_cast<const uint4*>(h);
    }
}

// saved activations -> the dW GEMM's A operand.  grid = (max F / 128, row chunks, layer), 256 threads; a thread writes 16-byte core-matrix rows
// (8 consecutive minibatch rows of one feature)
__global__ void __launch_bounds__(256) dm_learn_transpose_kernel(LearnTransposeParams P) {
    // the layer's fields without a dynamic index into the parameter arrays (which would copy them to local memory)
    const int l = blockIdx.z;
    auto pick = [l](auto a, auto b, auto c) { return l == 0 ? a : l == 1 ? b : c; };
    const int F = pick(P.F[0], P.F[1], P.F[2]), ones = pick(P.ones[0], P.ones[1], P.ones[2]), src_nc = pick(P.src_nc[0], P.src_nc[1], P.src_nc[2]);
    const __half* src = pick(P.src[0], P.src[1], P.src[2]);
    if (static_cast<int>(blockIdx.x) * 128 >= F) return;
    __half* dst = pick(P.dst[0], P.dst[1], P.dst[2]) + (static_cast<size_t>(blockIdx.x) * P.row_chunks + blockIdx.y) * kMlpATile;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int u = threadIdx.x + i * 256, k8 = u >> 7, fl = u & 127;
        const int f = blockIdx.x * 128 + fl, b0 = blockIdx.y * 64 + k8 * 8;
        __align__(16) __half h[8];
        if (f == ones) {
#pragma unroll
            for (int e = 0; e < 8; ++e) h[e] = __float2half_rn(1.f);
        } else if (f < src_nc * 64) {
            const __half* s = src + (static_cast<size_t>(b0 >> 7) * src_nc + (f >> 6)) * kMlpATile + ((((f & 63) >> 3) * 16 + ((b0 & 127) >> 3)) * 64 + (f & 7));
#pragma unroll
            for (int e = 0; e < 8; ++e) h[e] = s[e * 8];
        } else {
#pragma unroll
            for (int e = 0; e < 8; ++e) h[e] = __float2half_rn(0.f);
        }
        *reinterpret_cast<uint4*>(dst + ((k8 * 16 + (fl >> 3)) * 64 + (fl & 7) * 8)) = *reinterpret_cast<const uint4*>(h);
    }
}

// hi + lo fp16 parts of a head's dY g.  |g| <= 65504 splits as __float2half_rn gives it; past fp16's range hi saturates at +-65504 and lo
// carries the rest (|g| beyond 131008 saturates there), so such a row reaches the backward GEMMs finite instead of as inf + -inf = NaN.  NaN
// stays NaN
__device__ __forceinline__ void head_split(float g, __half& hi, __half& lo) {
    constexpr float kHalfMax = 65504.f;
    const auto sat = [](float v) { return fabsf(v) > kHalfMax ? copysignf(kHalfMax, v) : v; };
    hi = __float2half_rn(sat(g));
    lo = __float2half_rn(sat(g - __half2float(hi)));
}

// the per-row loss gradients w.r.t. the normalised output; one thread per row, grid = m tiles
template <bool ACTOR>
__device__ __forceinline__ void learn_head(const LearnHeadParams& P) {
    __shared__ float red[3][kLearnRows];
    const int tid = threadIdx.x, row = blockIdx.x * kLearnRows + tid;
    __half* dya = P.dy_a + static_cast<size_t>(blockIdx.x) * 2 * kMlpATile;
    __half* dyb = P.dy_b + static_cast<size_t>(row >> 6) * 2 * 64 * 64;
    const int k = row & 63;
    float part[3] = {0.f, 0.f, 0.f};
    float coef = 0.f;
    const int64_t s = row < P.M ? P.idx[row] : 0;
    const float* out = P.out + static_cast<size_t>(row) * P.out_dim;
    if constexpr (ACTOR) {
        if (row < P.M) {
            // logp of the normalised action under N(mu, sigma); the clipped surrogate's gradient rule as TF takes it: tf.minimum passes the gradient
            // to the unclipped term on ties, tf.clip_by_value passes it inside [1 - eps, 1 + eps]
            // sum_j (-z_j^2 / 2 - log sigma_j - log(2 pi) / 2), z = (a - mu) / sigma with IEEE division whatever the build's flags.  The sum is
            // taken in fp64: its terms add up to |logp| ~ 1e2 for 28 actions at sigma 0.05, where one fp32 ulp (~8e-6) is already the
            // ratio's whole error budget
            double lp = 0.0;
            for (int j = 0; j < P.out_dim; ++j) {
                const float z = __fdiv_rn(P.actions[s * P.out_dim + j] - out[j], expf(P.logstd[j]));
                lp += static_cast<double>(-0.5f * z * z) - static_cast<double>(P.logstd[j]) - 0.91893853320467274;
            }
            const float ratio = expf(static_cast<float>(lp - static_cast<double>(P.old_logp[s]))), adv = P.adv[s];
            if (P.ratio) P.ratio[row] = ratio;
            const float rc = fminf(fmaxf(ratio, 1.f - P.ratio_clip), 1.f + P.ratio_clip);
            const float l0 = adv * ratio, l1 = adv * rc;
            const bool active = l0 <= l1 || (ratio >= 1.f - P.ratio_clip && ratio <= 1.f + P.ratio_clip);
            coef = active ? -adv * ratio : 0.f;
            part[0] = -fminf(l0, l1);
            part[2] = fabsf(ratio - 1.f) > P.ratio_clip ? 1.f : 0.f;
        }
    }
    for (int j = 0; j < 64; ++j) {
        float g = 0.f;
        if (row < P.M && j < P.out_dim) {
            if constexpr (ACTOR) {
                const float mu = out[j];
                const float vmin = fminf(mu - P.bound_min[j], 0.f), vmax = fmaxf(mu - P.bound_max[j], 0.f);
                g = coef * (P.actions[s * P.out_dim + j] - mu) * expf(-2.f * P.logstd[j]) + vmin + vmax;
                part[1] += 0.5f * (vmin * vmin + vmax * vmax);
            } else {
                const float d = out[0] - P.targets[s];
                g = d;
                part[0] = 0.5f * d * d;
            }
        }
        __half hi, lo;
        head_split(g, hi, lo);
        const int oa = ((j >> 3) * 16 + (tid >> 3)) * 64 + (tid & 7) * 8 + (j & 7);
        dya[oa] = hi;
        dya[oa + kMlpATile] = lo;
        const int o = ((k >> 3) * 8 + (j >> 3)) * 64 + (j & 7) * 8 + (k & 7);
        dyb[o] = hi;
        dyb[o + 64 * 64] = lo;
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) red[i][tid] = part[i];
    __syncthreads();
    for (int w = kLearnRows / 2; w > 0; w >>= 1) {
        if (tid < w)
#pragma unroll
            for (int i = 0; i < 3; ++i) red[i][tid] += red[i][tid + w];
        __syncthreads();
    }
    if (tid < 3) P.partials[blockIdx.x * 3 + tid] = red[tid][0];
}
__global__ void __launch_bounds__(kLearnRows) dm_learn_actor_head_kernel(LearnHeadParams P) { learn_head<true>(P); }
__global__ void __launch_bounds__(kLearnRows) dm_learn_critic_head_kernel(LearnHeadParams P) { learn_head<false>(P); }

// one thread: the CTA partials in a fixed order, added to the running statistics.  Actor: stats[0] += |surrogate + bound loss| (the reference
// logs the absolute actor loss), stats[1] += clip fraction; critic: stats[0] += value loss
__global__ void dm_learn_stats_kernel(const float* partials, int ctas, float inv_rows, int actor, float* stats) {
    float s[3] = {0.f, 0.f, 0.f};
    for (int c = 0; c < ctas; ++c)
        for (int i = 0; i < 3; ++i) s[i] += partials[c * 3 + i];
    if (actor) {
        stats[0] += fabsf((s[0] + s[1]) * inv_rows);
        stats[1] += s[2] * inv_rows;
    } else {
        stats[0] += s[0] * inv_rows;
    }
}

// hi + lo operand-tile position of element (k, n) of a [K x N] B operand tiled with width BN and NC K-chunks (mlp_capi.cu: tile_weights)
__device__ __forceinline__ size_t learn_tile_off(int k, int n, int NC, int BN) {
    return (static_cast<size_t>(n / BN) * NC + (k >> 6)) * 2 * BN * 64 + ((((k & 63) >> 3) * (BN >> 3) + ((n % BN) >> 3)) * 64 + (n & 7) * 8 + (k & 7));
}
__device__ __forceinline__ void learn_put(__half* t, size_t o, int BN, float v) {
    const __half hi = __float2half_rn(v);
    t[o] = hi;
    t[o + static_cast<size_t>(BN) * 64] = __float2half_rn(v - __half2float(hi));
}

// grid = (ceil((in_dim + 1) / 256), out_dim), 256 threads: thread k of row n owns w[n][k], k == in_dim owns b[n]
__global__ void __launch_bounds__(256) dm_learn_layer_kernel(LearnLayerParams L) {
    const int k = blockIdx.x * 256 + threadIdx.x, n = blockIdx.y;
    if (k > L.in_dim) return;
    const bool bias = k == L.in_dim;
    float* p = bias ? L.b + n : L.w + static_cast<size_t>(n) * L.in_dim + k;
    float w = *p;
    if (L.acc_w) {
        float g = 0.f;
        for (int z = 0; z < L.splits; ++z) g += L.partial[(static_cast<size_t>(z) * L.Npad + n) * L.F + k];
        g *= L.inv_rows;
        if (!bias) g += L.wd * w;   // d/dw of wd sum ||W||^2 / 2 (PPOAgent._weight_decay_loss skips the biases)
        float* a = bias ? L.acc_b + n : L.acc_w + static_cast<size_t>(n) * L.in_dim + k;
        const float acc = L.mom * *a + g;
        *a = acc;
        w -= L.lr * acc;
        *p = w;
    }
    if (bias) {
        L.bias_pad[n] = w;
        return;
    }
    learn_put(L.tiles, learn_tile_off(k, n, L.NC, L.BN), L.BN, w);
    if (L.t_tiles) learn_put(L.t_tiles, learn_tile_off(n, k, L.t_NC, 128), 128, w);
}

// a plain handle's normaliser from device statistics: mean as is, std either inverted (the input normaliser keeps 1 / std, IEEE-rounded as
// dm_mlp_create's host division is) or as is (the output normaliser)
__global__ void __launch_bounds__(256) dm_learn_norm_kernel(const float* mean, const float* std_dev, int n, float* d_mean, float* d_std, int invert) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    d_mean[i] = mean[i];
    d_std[i] = invert ? __frcp_rn(std_dev[i]) : std_dev[i];
}

// ---- the AMP discriminator's minibatch step (R/learning/amp_agent.py: AMPAgent._build_losses, _disc_grad_penalty_loss; mlp_capi.cu:
// dm_learn_disc_step).  A step of `rows` agent and `rows` expert rows puts the agent rows at [0, rows) and the expert rows at [E, E + rows),
// E = pad128(rows), so every m tile holds one side only and the penalty's GEMMs address the expert tiles from tile E / 128 on.

// one thread per row, grid = 2E / 128.  Least-squares loss (Peng et al. 2021, eq. 8): 0.5 (0.5 mean (d_e - 1)^2 + 0.5 mean (d_a + 1)^2), so the
// gradient of the SUM over rows is 0.5 (d - 1) on an expert row and 0.5 (d + 1) on an agent row (1 / rows is applied by the optimiser)
__global__ void __launch_bounds__(kLearnRows) dm_learn_disc_head_kernel(LearnDiscHeadParams P) {
    __shared__ float red[3][kLearnRows];
    const int tid = threadIdx.x, row = blockIdx.x * kLearnRows + tid;
    const bool expert = row >= P.E;
    const int r = expert ? row - P.E : row;
    const bool real = r < P.rows;
    float g = 0.f, part[3] = {0.f, 0.f, 0.f};
    if (real) {
        const float d = P.out[row], e = d - (expert ? 1.f : -1.f);
        g = 0.5f * e;
        part[0] = e * e;
        part[1] = (expert ? d > 0.f : d < 0.f) ? 1.f : 0.f;
        part[2] = d;
    }
    __half* dya = P.dy_a + static_cast<size_t>(blockIdx.x) * 2 * kMlpATile;
    __half* dyb = P.dy_b + static_cast<size_t>(row >> 6) * 2 * 64 * 64;
    __half* sa = expert ? P.seed_a + static_cast<size_t>(blockIdx.x - P.E / kLearnRows) * 2 * kMlpATile : nullptr;
    __half* sb = expert ? P.seed_b + static_cast<size_t>(r >> 6) * 2 * 64 * 64 : nullptr;
    const int k = row & 63;
    const __half zero = __float2half_rn(0.f);
    for (int j = 0; j < 64; ++j) {
        const float v = j == 0 ? g : 0.f;
        const __half hi = __float2half_rn(v), lo = __float2half_rn(v - __half2float(hi));
        const int oa = ((j >> 3) * 16 + (tid >> 3)) * 64 + (tid & 7) * 8 + (j & 7);
        const int o = ((k >> 3) * 8 + (j >> 3)) * 64 + (j & 7) * 8 + (k & 7);
        dya[oa] = hi;
        dya[oa + kMlpATile] = lo;
        dyb[o] = hi;
        dyb[o + 64 * 64] = lo;
        if (expert) {
            sa[oa] = sb[o] = __float2half_rn(j == 0 && real ? 1.f : 0.f);
            sa[oa + kMlpATile] = sb[o + 64 * 64] = zero;
        }
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) red[i][tid] = part[i];
    __syncthreads();
    for (int w = kLearnRows / 2; w > 0; w >>= 1) {
        if (tid < w)
#pragma unroll
            for (int i = 0; i < 3; ++i) red[i][tid] += red[i][tid + w];
        __syncthreads();
    }
    if (tid < 3) P.partials[blockIdx.x * 3 + tid] = red[tid][0];
}

// ||g||^2 of every expert row, g = dd / dx the input gradient held as hi + lo operand tiles [E / 128][hi: NC, lo: NC][kMlpATile]; one thread
// per row (a thread reads 16-byte core-matrix rows: 8 consecutive inputs of its row), the CTA's sum in a fixed tree.  grid = E / 128
__global__ void __launch_bounds__(kLearnRows) dm_learn_disc_gp_kernel(const __half* g, int NC, float* partials) {
    __shared__ float red[kLearnRows];
    const int tid = threadIdx.x;
    const __half* base = g + static_cast<size_t>(blockIdx.x) * 2 * NC * kMlpATile;
    float s = 0.f;
    for (int c = 0; c < NC; ++c)
        for (int k8 = 0; k8 < 8; ++k8) {
            const size_t o = static_cast<size_t>(c) * kMlpATile + (k8 * 16 + (tid >> 3)) * 64 + (tid & 7) * 8;
            __align__(16) __half hi[8], lo[8];
            *reinterpret_cast<uint4*>(hi) = *reinterpret_cast<const uint4*>(base + o);
            *reinterpret_cast<uint4*>(lo) = *reinterpret_cast<const uint4*>(base + o + static_cast<size_t>(NC) * kMlpATile);
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const float v = __half2float(hi[e]) + __half2float(lo[e]);
                s += v * v;
            }
        }
    red[tid] = s;
    __syncthreads();
    for (int w = kLearnRows / 2; w > 0; w >>= 1) {
        if (tid < w) red[tid] += red[tid + w];
        __syncthreads();
    }
    if (tid == 0) partials[blockIdx.x] = red[0];
}

// one thread: the CTA partials in a fixed order (head CTAs [0, ctas / 2) hold agent rows, the rest expert rows), added to the running statistics:
// stats[0] += the least-squares loss, [1] += 0.5 mean ||g||^2 (unweighted), [2] += mean(d_e > 0), [3] += mean(d_a < 0), [4] += mean d_e,
// [5] += mean d_a
__global__ void dm_learn_disc_stats_kernel(const float* head, int ctas, const float* gp, int gp_ctas, float inv_rows, float* stats) {
    float a[3] = {0.f, 0.f, 0.f}, e[3] = {0.f, 0.f, 0.f}, q = 0.f;
    for (int c = 0; c < ctas; ++c)
        for (int i = 0; i < 3; ++i) (c < ctas / 2 ? a : e)[i] += head[c * 3 + i];
    for (int c = 0; c < gp_ctas; ++c) q += gp[c];
    stats[0] += 0.25f * (e[0] + a[0]) * inv_rows;
    stats[1] += 0.5f * q * inv_rows;
    stats[2] += e[1] * inv_rows;
    stats[3] += a[1] * inv_rows;
    stats[4] += e[2] * inv_rows;
    stats[5] += a[2] * inv_rows;
}

// dm_learn_layer_kernel with the penalty's partials and the logit regulariser: g = (sum dW + gp_w sum dW_pen) / rows + (wd + reg) w on the
// weights, (sum db) / rows on the biases; then the momentum step and the re-tiling
__global__ void __launch_bounds__(256) dm_learn_disc_layer_kernel(LearnDiscLayerParams D) {
    const LearnLayerParams& L = D.L;
    const int k = blockIdx.x * 256 + threadIdx.x, n = blockIdx.y;
    if (k > L.in_dim) return;
    const bool bias = k == L.in_dim;
    float* p = bias ? L.b + n : L.w + static_cast<size_t>(n) * L.in_dim + k;
    float w = *p;
    if (L.acc_w) {
        float g = 0.f;
        for (int z = 0; z < L.splits; ++z) g += L.partial[(static_cast<size_t>(z) * L.Npad + n) * L.F + k];
        if (!bias && D.pen) {
            float q = 0.f;
            for (int z = 0; z < D.pen_splits; ++z) q += D.pen[(static_cast<size_t>(z) * L.Npad + n) * D.pen_F + k];
            g += D.gp_w * q;
        }
        g *= L.inv_rows;
        if (!bias) g += (L.wd + D.reg) * w;
        float* a = bias ? L.acc_b + n : L.acc_w + static_cast<size_t>(n) * L.in_dim + k;
        const float acc = L.mom * *a + g;
        *a = acc;
        w -= L.lr * acc;
        *p = w;
    }
    if (bias) {
        L.bias_pad[n] = w;
        return;
    }
    learn_put(L.tiles, learn_tile_off(k, n, L.NC, L.BN), L.BN, w);
    if (L.t_tiles) learn_put(L.t_tiles, learn_tile_off(n, k, L.t_NC, 128), 128, w);
    if (D.p_tiles) learn_put(D.p_tiles, learn_tile_off(k, n, D.p_NC, 128), 128, w);
}

// ---- the step split in two for data-parallel training (dm_learn_*grad, dm_learn_*apply): the layer passes above, cut after the gradient's
// reduction over the step's rows.  Between the halves the callers sum the ranks' gradients.  The arithmetic is the layer passes', operation
// for operation; the intrinsics pin the rounding nvcc's contraction gives the fused kernels (an FMUL by 1 / rows, FFMAs for the penalty, the
// weight decay, the momentum and the step), so apply(grad(b), scale 1) reproduces the fused step bit for bit.

// the mean gradient of one parameter pair without its weight decay: g = (sum dW + gp_w sum dW_pen) / rows on the weights, (sum db) / rows on the
// biases, the split partials summed in dm_learn_layer_kernel's order.  D.pen null: the PPO networks.  grid as dm_learn_layer_kernel
__global__ void __launch_bounds__(256) dm_learn_pack_kernel(LearnDiscLayerParams D, LearnGradParams G) {
    const LearnLayerParams& L = D.L;
    const int k = blockIdx.x * 256 + threadIdx.x, n = blockIdx.y;
    if (k > L.in_dim) return;
    const bool bias = k == L.in_dim;
    float g = 0.f;
    for (int z = 0; z < L.splits; ++z) g += L.partial[(static_cast<size_t>(z) * L.Npad + n) * L.F + k];
    if (!bias && D.pen) {
        float q = 0.f;
        for (int z = 0; z < D.pen_splits; ++z) q += D.pen[(static_cast<size_t>(z) * L.Npad + n) * D.pen_F + k];
        g = __fmaf_rn(D.gp_w, q, g);
    }
    g = __fmul_rn(g, L.inv_rows);
    if (bias) G.b[n] = g;
    else G.w[static_cast<size_t>(n) * L.in_dim + k] = g;
}

// the optimiser half: g = scale G + (wd + reg) w on the weights, scale G on the biases; then the momentum step and the re-tiling of
// dm_learn_disc_layer_kernel (D.reg = 0 and no p_tiles: dm_learn_layer_kernel's)
__global__ void __launch_bounds__(256) dm_learn_apply_kernel(LearnDiscLayerParams D, LearnGradParams G) {
    const LearnLayerParams& L = D.L;
    const int k = blockIdx.x * 256 + threadIdx.x, n = blockIdx.y;
    if (k > L.in_dim) return;
    const bool bias = k == L.in_dim;
    float* p = bias ? L.b + n : L.w + static_cast<size_t>(n) * L.in_dim + k;
    float w = *p;
    float g = __fmul_rn(bias ? G.b[n] : G.w[static_cast<size_t>(n) * L.in_dim + k], G.scale);
    if (!bias) g = __fmaf_rn(__fadd_rn(L.wd, D.reg), w, g);
    float* a = bias ? L.acc_b + n : L.acc_w + static_cast<size_t>(n) * L.in_dim + k;
    const float acc = __fmaf_rn(L.mom, *a, g);
    *a = acc;
    w = __fmaf_rn(-L.lr, acc, w);
    *p = w;
    if (bias) {
        L.bias_pad[n] = w;
        return;
    }
    learn_put(L.tiles, learn_tile_off(k, n, L.NC, L.BN), L.BN, w);
    if (L.t_tiles) learn_put(L.t_tiles, learn_tile_off(n, k, L.t_NC, 128), 128, w);
    if (D.p_tiles) learn_put(D.p_tiles, learn_tile_off(k, n, D.p_NC, 128), 128, w);
}

}  // namespace dmk
