// Policy network of the batched rollout (SURVEY.md 8(f) rank 1): the actor of the reference's PPO / AMP agents,
//   a = un-normalise( W2^T relu( W1^T relu( W0^T normalise(s) + b0 ) + b1 ) + b2 )        (R/learning/nets/fc_2layers_1024units.py,
//   R/learning/pg_agent.py:140-160, R/learning/normalizer.py), 227 -> 1024 -> 512 -> 28 for humanoid3d,
// as one operand-preparation launch + three launches of one sm_90a GEMM kernel built on Hopper's warpgroup tensor-core instructions:
//   * wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 with both operands read from shared memory through matrix descriptors: each of the
//     two warpgroups of a CTA owns 64 of its 128 rows and accumulates BN columns (one 64-column accumulator per 64 columns) in registers (fp32),
//   * BOTH operands live in global memory already tiled in the shared-memory operand layout (canonical K-major, no swizzle: 8 x 16-byte core
//     matrices): the weights are tiled once on the host, the activations are written in that layout by the producing launch (the preparation
//     kernel for the observations, the previous layer's epilogue otherwise).  A K-chunk of either operand is therefore ONE contiguous block
//     that the TMA unit brings in as a bulk copy (cp.async.bulk ... mbarrier::complete_tx),
//   * 2-stage full / empty mbarrier pipeline (2 x 48 KB of shared memory: two CTAs per SM, so one CTA's copies overlap the other's MMAs):
//     thread 0 issues the bulk copies of chunk c + 2 once every thread has released the stage of chunk c,
//   * every weight is carried as fp16 hi + fp16 lo (w = hi + lo to 2^-22): two MMAs per K-step make the weights exact to fp32 level, so the only
//     rounding beyond the fp32 reference is the fp16 rounding of the activations (measured action error < 1e-3, tests/test_mlp_gpu.py),
//   * epilogue straight from the accumulator registers: bias, ReLU, fp16 pairs into the next layer's operand tiles (a warp's store covers one
//     128-byte core matrix); the last layer adds the exploration noise and un-normalises into the DeepMimic action layout (fp32).
// The gated actor of the AMP task scenes (R/learning/nets/fc_2layers_gated_1024units.py) reuses these pieces: the preparation kernel also writes
// the normalised goal (into the trunk's columns after the state, and alone as the gate trunk's operand), the gate trunk and both gate hidden
// layers are launches of the 128-column kernel, and each trunk layer is a GATED instantiation whose pipeline appends the gate's scale and bias
// chunks (DESIGN.md section 8).
// This is the one dense contraction next to the hot path (the simulation itself has none); it replaces cuBLAS / eager torch in the rollout shim.
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cstdint>

#include "dm_mlp.cuh"

namespace dmk {

constexpr int kMlpThreads = 128;     // operand-preparation kernel
constexpr int kMlpGemmThreads = 256; // GEMM kernel: two warpgroups, warpgroup g owns rows [64 g, 64 g + 64) of the CTA tile
constexpr int kMlpStages = 2;

// The modes of the backward GEMMs of the PPO learner (MlpGradParams): same pipeline, other operands and epilogues:
//   GRAD_X  dH = (dY W^T) * 1[H > 0]: A = dY in operand layout as hi + lo chunks (K = twice this layer's padded outputs), B = W^T as hi + lo
//           tiles (N = its padded inputs), so both operands are exact to fp32 level (a minibatch's gradient is a sum of per-row terms that
//           largely cancel, which magnifies fp16 rounding of dY); the epilogue masks with the saved forward activation tile and writes dH as the
//           next dX GEMM's A operand and, as hi + lo, as the dW GEMM's B operand
//   GRAD_W  dW = X^T dY: A = the layer's input activations transposed (M = padded inputs + the ones feature whose dW row is db), B = dY as
//           hi + lo (K = minibatch rows); K is split over row-chunk ranges (blockIdx.z) and each split writes its fp32 partial product
//   GRAD_XA the AMP discriminator's gradient-penalty chain: the GRAD_X pipeline (B = W^T, or a layer's forward tiles for a product W x), the
//           mask only where mask_tiles is given, and dH written as the next GEMM's A operand only (dy_a), never as a dW operand
//   GRAD_XG the dX GEMM into a gated layer's output h (dm_learn_gated_step): p = dh 1[h > 0], then dz = a p written as GRAD_X writes dH, and
//           ds = b p, dt = p (MlpGateParams) as hi + lo A operands of the gate's dX GEMM and B operands of the gate's dW GEMM
//   SAVE    not a backward GEMM: the gated forward epilogue of the learner, which also writes the factors a = 2 sigmoid(s) and
//           b = 2 sigmoid(s) (1 - sigmoid(s)) z (z = acc + bias) of every row and unit, so that the backward uses the forward's own sigmoid
enum { kGradNone = 0, kGradX = 1, kGradW = 2, kGradXA = 3, kGradXG = 4, kGradSave = 5 };

namespace {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count)); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory"); }
// bounded spin: a protocol error traps (the launch fails with an error) instead of hanging the GPU
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    for (uint32_t spin = 0;; ++spin) {
        uint32_t ok;
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.b32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(addr), "r"(parity) : "memory");
        if (ok) return;
        if (spin > (1u << 26)) __trap();
    }
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// wgmma shared-memory matrix descriptor, canonical K-major layout without swizzle (layout type 0):
//   core matrix = 8 rows x 16 bytes, rows 16 bytes apart; LBO = bytes between the two 16-byte K slices, SBO = bytes between 8-row groups
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return static_cast<uint64_t>((saddr >> 4) & 0x3FFFu) | (static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16) | (static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32);
}
// D[64 x 64] (+)= A[64 x 16] B[16 x 64]: fp16 x fp16 -> fp32, both operands K-major in shared memory, D in 32 registers per thread
__device__ __forceinline__ void wgmma_64x64x16(float* d, uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}
// keeps the compiler from moving accesses of the accumulator registers across the asynchronous MMAs
__device__ __forceinline__ void fence_acc(float& r) { asm volatile("" : "+f"(r)::"memory"); }

}  // namespace

// Observations -> normalised, clipped fp16 activations in operand layout.  grid = (m tiles, K chunks [+ 1 for the goal's own tile]), 128 threads:
// 8 consecutive threads cover 64 consecutive inputs of one row (coalesced 256-byte reads), a thread writes one 16-byte core-matrix row.
template <bool GOAL>
__device__ __forceinline__ void mlp_prep(const MlpPrepParams& P) {
    const int m0 = blockIdx.x * kMlpBM;
    const bool gate = GOAL && blockIdx.y == P.NC;   // the gate trunk's operand: the normalised goal from column 0
    const int c = gate ? 0 : blockIdx.y;
    __half* tile = gate ? P.g_tiles + static_cast<size_t>(blockIdx.x) * kMlpATile : P.tiles + (static_cast<size_t>(blockIdx.x) * P.NC + c) * kMlpATile;
#pragma unroll
    for (int i = 0; i < (kMlpBM * 8) / kMlpThreads; ++i) {
        const int u = threadIdx.x + i * kMlpThreads, row = u >> 3, k8 = u & 7;
        const int grow = m0 + row, k = c * kMlpBK + k8 * 8;
        __align__(16) __half h[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            float x = 0.f;
            if (grow < P.M && !gate && k + e < P.in_dim) {
                x = (P.obs[static_cast<size_t>(grow) * P.in_dim + k + e] - P.in_mean[k + e]) * P.in_istd[k + e];
                x = fminf(fmaxf(x, -P.in_clip), P.in_clip);
            } else if (GOAL && grow < P.M) {
                const int j = gate ? k + e : k + e - P.in_dim;
                if (j < P.goal_dim) {
                    x = (P.goal[static_cast<size_t>(grow) * P.goal_dim + j] - P.g_mean[j]) * P.g_istd[j];
                    x = fminf(fmaxf(x, -P.g_clip), P.g_clip);
                }
            }
            h[e] = __float2half_rn(x);
        }
        *reinterpret_cast<uint4*>(tile + ((k8 * (kMlpBM / 8) + (row >> 3)) * 64 + (row & 7) * 8)) = *reinterpret_cast<const uint4*>(h);
    }
}

__global__ void __launch_bounds__(kMlpThreads) dm_mlp_prep_kernel(MlpPrepParams P) { mlp_prep<false>(P); }
// [normalised state | normalised goal] trunk tiles, and the normalised goal's own tile
__global__ void __launch_bounds__(kMlpThreads) dm_mlp_gated_prep_kernel(MlpPrepParams P) { mlp_prep<true>(P); }

// C[M x N] = act(A[M x K] W + b); grid = (M / 128, N / BN), block = 256 threads (two warpgroups),
// dynamic shared memory = 2 stages x (A 16 KB + W hi/lo 2 x BN x 128 B) + 1 KB (barriers).
// GATED (a hidden layer of the gated actor): two more pipeline chunks after the K loop (MlpGemmParams::gate_tiles) accumulate the gate's scale
// and bias pre-activations in registers of their own; with BN = 64 that is 3 x 32 accumulator registers per thread.
// STYLE (the discriminator's one-unit logit head): the last layer's epilogue writes the style reward instead of actions.
// GRAD (the learner's backward GEMMs, MlpGradParams): kGradX / kGradW epilogues; kGradW also takes its K range from blockIdx.z.
// Q (MlpGateParams): kGradXG, and kGradSave on a GATED layer.
template <int BN, bool LAST, bool GATED, bool STYLE = false, int GRAD = kGradNone>
__device__ __forceinline__ void mlp_gemm(const MlpGemmParams& P, const MlpStyleParams* S = nullptr, const MlpGradParams* G = nullptr,
                                         const MlpGateParams* Q = nullptr) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    constexpr int kABytes = kMlpATile * 2;               // 16 KB
    constexpr int kWBytes = 2 * BN * kMlpBK * 2;         // hi + lo
    constexpr int kStage = kABytes + kWBytes;
    constexpr int NH = BN / 64;                          // 64-column accumulators per warpgroup
    static_assert(!GATED || (!LAST && NH == 1), "the gated epilogue is written for one 64-column accumulator of a hidden layer");
    static_assert(!STYLE || (LAST && !GATED && NH == 1), "the style-reward epilogue is written for one 64-column accumulator of the last layer");
    uint64_t* bar_full = reinterpret_cast<uint64_t*>(smem_raw + kMlpStages * kStage);   // [stages] both operands of the stage have landed
    uint64_t* bar_empty = bar_full + kMlpStages;                                         // [stages] every thread's MMAs reading the stage have completed
    const int tid = threadIdx.x, wg = tid >> 7, wtid = tid & 127;
    const int mt = blockIdx.x, m0 = mt * kMlpBM, nt = blockIdx.y, n0 = nt * BN;
    static_assert(GRAD == kGradNone || (!LAST && GATED == (GRAD == kGradSave) && !STYLE), "the gradient epilogues replace the hidden-layer epilogue");
    // kGradW: this split's row chunks [c0, c0 + NC) of the KC chunks every m / n tile holds
    // kGradX: A is dY as hi chunks then lo chunks (2 K / 64 chunks per m tile), each against the same W^T chunk: dY exact to fp32 level
    constexpr bool kDyHiLo = GRAD == kGradX || GRAD == kGradXA || GRAD == kGradXG;
    const int KW = GRAD == kGradW ? G->row_chunks : P.K / kMlpBK;   // K chunks per n tile of B
    const int KC = kDyHiLo ? 2 * KW : KW;                           // K chunks per m tile of A
    const int c0 = GRAD == kGradW ? static_cast<int>(blockIdx.z) * G->chunks_per_split : 0;
    const int NC = GRAD == kGradW ? min(G->chunks_per_split, KC - c0) : KC;
    const int NT = GATED ? NC + 2 : NC;                  // pipeline chunks: the K loop, then the gate's scale and bias chunks
    const __half* a_src = P.a_tiles + (static_cast<size_t>(mt) * KC + c0) * kMlpATile;
    const __half* w_src = P.w_tiles + (static_cast<size_t>(nt) * KW + c0) * (kWBytes / 2);
    // one bulk copy per operand and K-chunk (both are contiguous blocks in operand layout)
    auto load = [&](int c) {
        const int s = c % kMlpStages;
        uint8_t* sA = smem_raw + s * kStage;
        mbar_expect_tx(&bar_full[s], kStage);
        if (GATED && c >= NC) {
            bulk_g2s(sA, P.gate_tiles + static_cast<size_t>(mt) * P.gate_stride, kABytes, &bar_full[s]);
            bulk_g2s(sA + kABytes, (c == NC ? P.ws_tiles : P.wb_tiles) + static_cast<size_t>(nt) * (kWBytes / 2), kWBytes, &bar_full[s]);
            return;
        }
        bulk_g2s(sA, a_src + static_cast<size_t>(c) * kMlpATile, kABytes, &bar_full[s]);
        bulk_g2s(sA + kABytes, w_src + static_cast<size_t>(kDyHiLo ? c % KW : c) * (kWBytes / 2), kWBytes, &bar_full[s]);
    };

    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < kMlpStages; ++s) { mbar_init(&bar_full[s], 1); mbar_init(&bar_empty[s], kMlpGemmThreads); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        for (int c = 0; c < NT && c < kMlpStages; ++c) load(c);
    }
    __syncthreads();

    float acc[NH][32], acc_s[NH][32], acc_b[NH][32];     // acc_s / acc_b: GATED only
#pragma unroll
    for (int h = 0; h < NH; ++h)
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[h][i] = acc_s[h][i] = acc_b[h][i] = 0.f;
    constexpr uint32_t kALbo = (kMlpBM / 8) * 128, kBLbo = (BN / 8) * 128;
    // MMAs of pipeline chunk c into d, then release its stage and refill it with chunk c + 2
    auto mma_chunk = [&](int c, float (&d)[NH][32]) {
        const int s = c % kMlpStages;
        mbar_wait(&bar_full[s], (c / kMlpStages) & 1);
        // this warpgroup's 64 rows start 8 row groups (1 KB) into each K slice of the A tile; columns [64 h, 64 h + 64) likewise in W
        const uint32_t a0 = smem_u32(smem_raw + s * kStage) + wg * 1024, b0 = smem_u32(smem_raw + s * kStage + kABytes);
#pragma unroll
        for (int h = 0; h < NH; ++h)
#pragma unroll
            for (int i = 0; i < 32; ++i) fence_acc(d[h][i]);
        asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
        for (int j = 0; j < kMlpBK / 16; ++j) {
            const uint64_t ad = wgmma_desc(a0 + j * 2 * kALbo, kALbo, 128);
#pragma unroll
            for (int h = 0; h < NH; ++h) {
                const uint32_t bh = b0 + h * 1024 + j * 2 * kBLbo;
                wgmma_64x64x16(d[h], ad, wgmma_desc(bh, kBLbo, 128), 1u);
                wgmma_64x64x16(d[h], ad, wgmma_desc(bh + BN * kMlpBK * 2, kBLbo, 128), 1u);
            }
        }
        asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
        asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
#pragma unroll
        for (int h = 0; h < NH; ++h)
#pragma unroll
            for (int i = 0; i < 32; ++i) fence_acc(d[h][i]);
        mbar_arrive(&bar_empty[s]);
        if (tid == 0 && c + kMlpStages < NT) {
            mbar_wait(&bar_empty[s], (c / kMlpStages) & 1);
            load(c + kMlpStages);
        }
        __syncwarp();
    };
#pragma unroll 1
    for (int c = 0; c < NC; ++c) mma_chunk(c, acc);
    if constexpr (GATED) {
        mma_chunk(NC, acc_s);
        mma_chunk(NC + 1, acc_b);
    }

    // ---- epilogue from the accumulator fragments: register i of accumulator h holds row 16 w + lane / 4 (+ 8 for i & 2) of the warpgroup's
    //      64 rows and column 64 h + 8 (i / 4) + 2 (lane % 4) + (i & 1)
    const int warp = wtid >> 5, lane = wtid & 31;
#pragma unroll
    for (int h = 0; h < NH; ++h) {
#pragma unroll
        for (int q = 0; q < 16; ++q) {
            const int r = wg * 64 + warp * 16 + (lane >> 2) + 8 * (q & 1), row = m0 + r;
            const int n = n0 + h * 64 + 8 * (q >> 1) + 2 * (lane & 3);
            const int i0 = 4 * (q >> 1) + 2 * (q & 1);
            const float v0 = acc[h][i0], v1 = acc[h][i0 + 1];
            if constexpr (GRAD == kGradW) {
                // row = input feature, n = output unit: the partial sum of this split in the parameter's [out x in] order (every row of the
                // padded M is written; the optimiser reads the real ones)
                float* out = G->partial + static_cast<size_t>(blockIdx.z) * P.N * P.M;
                out[static_cast<size_t>(n) * P.M + row] = v0;
                out[static_cast<size_t>(n + 1) * P.M + row] = v1;
            } else if constexpr (GRAD == kGradX) {
                // ReLU mask from the saved fp16 activation: a pre-activation in (0, 2^-25) rounded to 0 there and is masked (within tolerance)
                const size_t in_tile = (((n & 63) >> 3) * (kMlpBM / 8) + (r >> 3)) * 64 + (r & 7) * 8 + (n & 7);
                const __half2 hact = *reinterpret_cast<const __half2*>(G->mask_tiles + (static_cast<size_t>(mt) * (P.N >> 6) + (n >> 6)) * kMlpATile + in_tile);
                const float d0 = __low2float(hact) > 0.f ? v0 : 0.f, d1 = __high2float(hact) > 0.f ? v1 : 0.f;
                if (G->dy_a) {
                    // the next dX GEMM's A: hi in chunk n / 64, lo in chunk N / 64 + n / 64 of the m tile's 2 N / 64 chunks
                    __half* t = G->dy_a + (static_cast<size_t>(mt) * 2 * (P.N >> 6) + (n >> 6)) * kMlpATile + in_tile;
                    const __half2 hi = __floats2half2_rn(d0, d1);
                    *reinterpret_cast<__half2*>(t) = hi;
                    *reinterpret_cast<__half2*>(t + static_cast<size_t>(P.N >> 6) * kMlpATile) = __floats2half2_rn(d0 - __low2float(hi), d1 - __high2float(hi));
                }
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int ne = n + e, k = row & 63;
                    const float d = e ? d1 : d0;
                    const __half hi = __float2half_rn(d);
                    __half* t = G->dy_b + (static_cast<size_t>(ne >> 7) * G->row_chunks + (row >> 6)) * 2 * 128 * kMlpBK +
                                (((k >> 3) * 16 + ((ne & 127) >> 3)) * 64 + (ne & 7) * 8 + (k & 7));
                    t[0] = hi;
                    t[128 * kMlpBK] = __float2half_rn(d - __half2float(hi));
                }
            } else if constexpr (GRAD == kGradXA) {
                const size_t in_tile = (((n & 63) >> 3) * (kMlpBM / 8) + (r >> 3)) * 64 + (r & 7) * 8 + (n & 7);
                float d0 = v0, d1 = v1;
                if (G->mask_tiles) {
                    const __half2 hact = *reinterpret_cast<const __half2*>(G->mask_tiles + (static_cast<size_t>(mt) * (P.N >> 6) + (n >> 6)) * kMlpATile + in_tile);
                    d0 = __low2float(hact) > 0.f ? v0 : 0.f;
                    d1 = __high2float(hact) > 0.f ? v1 : 0.f;
                }
                __half* t = G->dy_a + (static_cast<size_t>(mt) * 2 * (P.N >> 6) + (n >> 6)) * kMlpATile + in_tile;
                const __half2 hi = __floats2half2_rn(d0, d1);
                *reinterpret_cast<__half2*>(t) = hi;
                *reinterpret_cast<__half2*>(t + static_cast<size_t>(P.N >> 6) * kMlpATile) = __floats2half2_rn(d0 - __low2float(hi), d1 - __high2float(hi));
            } else if constexpr (GRAD == kGradXG) {
                const size_t in_tile = (((n & 63) >> 3) * (kMlpBM / 8) + (r >> 3)) * 64 + (r & 7) * 8 + (n & 7);
                const __half2 hact = *reinterpret_cast<const __half2*>(G->mask_tiles + (static_cast<size_t>(mt) * (P.N >> 6) + (n >> 6)) * kMlpATile + in_tile);
                const float p0 = __low2float(hact) > 0.f ? v0 : 0.f, p1 = __high2float(hact) > 0.f ? v1 : 0.f;
                const size_t o = static_cast<size_t>(row) * P.N + n;
                const float2 fa = *reinterpret_cast<const float2*>(Q->fa + o), fb = *reinterpret_cast<const float2*>(Q->fb + o);
                const float dz[2] = {fa.x * p0, fa.y * p1}, ds[2] = {fb.x * p0, fb.y * p1}, dt[2] = {p0, p1};
                // hi at t, lo `lo` halves further
                auto put_a = [&](__half* t, const float* d, size_t lo) {
                    const __half2 hi = __floats2half2_rn(d[0], d[1]);
                    *reinterpret_cast<__half2*>(t) = hi;
                    *reinterpret_cast<__half2*>(t + lo) = __floats2half2_rn(d[0] - __low2float(hi), d[1] - __high2float(hi));
                };
                // element (row, ne) of a dW GEMM's B operand [N' / 128][row_chunks][hi | lo][128 x 64]
                auto put_b = [&](__half* base, int ne, float d) {
                    const int k = row & 63;
                    const __half hi = __float2half_rn(d);
                    __half* t = base + (static_cast<size_t>(ne >> 7) * G->row_chunks + (row >> 6)) * 2 * 128 * kMlpBK +
                                (((k >> 3) * 16 + ((ne & 127) >> 3)) * 64 + (ne & 7) * 8 + (k & 7));
                    t[0] = hi;
                    t[128 * kMlpBK] = __float2half_rn(d - __half2float(hi));
                };
                if (G->dy_a) put_a(G->dy_a + (static_cast<size_t>(mt) * 2 * (P.N >> 6) + (n >> 6)) * kMlpATile + in_tile, dz, static_cast<size_t>(P.N >> 6) * kMlpATile);
                __half* sa = Q->st_a + (static_cast<size_t>(mt) * 2 * Q->st_nc + (n >> 6)) * kMlpATile + in_tile;
                put_a(sa + static_cast<size_t>(Q->s_chunk) * kMlpATile, ds, static_cast<size_t>(Q->st_nc) * kMlpATile);
                put_a(sa + static_cast<size_t>(Q->t_chunk) * kMlpATile, dt, static_cast<size_t>(Q->st_nc) * kMlpATile);
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    put_b(G->dy_b, n + e, dz[e]);
                    put_b(Q->st_b, n + e, ds[e]);
                    put_b(Q->st_b, P.N + n + e, dt[e]);
                }
            } else if constexpr (STYLE) {
                // the logit is column 0 (the tile's other 63 columns are padding): one thread per row holds it and writes every output of that row
                if (row < P.M && n == 0) {
                    const float d = v0 + P.bias[0], e = 1.f - d;
                    const float style = fmaxf(0.f, 1.f - 0.25f * e * e);
                    S->reward[row] = S->task_reward ? (1.f - S->task_lerp) * style + S->task_lerp * S->task_reward[row] : style;
                    if (S->logit) S->logit[row] = d;
                    if (S->style) S->style[row] = style;
                }
            } else if constexpr (LAST) {
                if (row < P.M) {
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int ne = n + e;
                        if (ne < P.out_dim) {
                            float a = (e ? v1 : v0) + P.bias[ne];
                            if (P.noise) a += P.noise[static_cast<size_t>(row) * P.out_dim + ne];
                            P.actions[static_cast<size_t>(row) * P.out_dim + ne] = a * P.out_std[ne] + P.out_mean[ne];
                        }
                    }
                }
            } else {
                // next layer's operand tiles: K index = this layer's column; rows past M carry relu(bias) (never read back as results)
                __half2 hv;
                if constexpr (GATED) {
                    float fa[2], fb[2];   // kGradSave: the backward's factors
                    auto gated = [&](float v, int i, int ne, int e) {
                        const float scale = 2.f / (1.f + __expf(-(acc_s[h][i] + P.bias_s[ne])));
                        const float z = v + P.bias[ne];
                        fa[e] = scale;
                        fb[e] = scale * (1.f - 0.5f * scale) * z;
                        return fmaxf(scale * z + acc_b[h][i] + P.bias_b[ne], 0.f);
                    };
                    hv = __floats2half2_rn(gated(v0, i0, n, 0), gated(v1, i0 + 1, n + 1, 1));
                    if constexpr (GRAD == kGradSave) {
                        const size_t o = static_cast<size_t>(row) * P.N + n;
                        *reinterpret_cast<float2*>(Q->fa + o) = make_float2(fa[0], fa[1]);
                        *reinterpret_cast<float2*>(Q->fb + o) = make_float2(fb[0], fb[1]);
                    }
                } else {
                    hv = __floats2half2_rn(fmaxf(v0 + P.bias[n], 0.f), fmaxf(v1 + P.bias[n + 1], 0.f));
                }
                __half* tile = P.out_tiles + (static_cast<size_t>(mt) * (P.N >> 6) + (n >> 6)) * kMlpATile;
                *reinterpret_cast<__half2*>(tile + ((((n & 63) >> 3) * (kMlpBM / 8) + (r >> 3)) * 64 + (r & 7) * 8 + (n & 7))) = hv;
            }
        }
    }
}

template <int BN, bool LAST>
__global__ void __launch_bounds__(kMlpGemmThreads, 2) dm_mlp_gemm_kernel(MlpGemmParams P) { mlp_gemm<BN, LAST, false>(P); }
// a hidden layer of the gated actor, 64-column tiles
__global__ void __launch_bounds__(kMlpGemmThreads, 2) dm_mlp_gated_gemm_kernel(MlpGemmParams P) { mlp_gemm<64, false, true>(P); }
// the discriminator's logit head with the style-reward epilogue (AMP, Peng et al. 2021, eq. 7), 64-column tile
__global__ void __launch_bounds__(kMlpGemmThreads, 2) dm_mlp_style_reward_kernel(MlpGemmParams P, MlpStyleParams S) { mlp_gemm<64, true, false, true>(P, &S); }

// the PPO learner's backward GEMMs (MlpGradParams): dX of a hidden layer (128-column tiles) and the split-K dW (BN = 128, or 64 for an output
// layer of up to 64 units)
__global__ void __launch_bounds__(kMlpGemmThreads, 2) dm_mlp_grad_x_kernel(MlpGemmParams P, MlpGradParams G) { mlp_gemm<128, false, false, false, kGradX>(P, nullptr, &G); }
template <int BN>
__global__ void __launch_bounds__(kMlpGemmThreads, 2) dm_mlp_grad_w_kernel(MlpGemmParams P, MlpGradParams G) { mlp_gemm<BN, false, false, false, kGradW>(P, nullptr, &G); }
template __global__ void dm_mlp_grad_w_kernel<128>(MlpGemmParams, MlpGradParams);
template __global__ void dm_mlp_grad_w_kernel<64>(MlpGemmParams, MlpGradParams);
// the AMP discriminator's gradient-penalty products (GRAD_XA, mlp_capi.cu: dm_learn_disc_step), 128-column tiles
__global__ void __launch_bounds__(kMlpGemmThreads, 2) dm_mlp_grad_xa_kernel(MlpGemmParams P, MlpGradParams G) { mlp_gemm<128, false, false, false, kGradXA>(P, nullptr, &G); }
// the gated PPO learner (mlp_capi.cu: dm_learn_gated_step): a gated trunk layer's forward that saves the backward's factors (64-column tiles,
// as dm_mlp_gated_gemm_kernel), and the dX GEMM into a gated layer's output (GRAD_XG, 128-column tiles)
__global__ void __launch_bounds__(kMlpGemmThreads, 2) dm_mlp_gated_save_kernel(MlpGemmParams P, MlpGateParams Q) { mlp_gemm<64, false, true, false, kGradSave>(P, nullptr, nullptr, &Q); }
__global__ void __launch_bounds__(kMlpGemmThreads, 2) dm_mlp_grad_xg_kernel(MlpGemmParams P, MlpGradParams G, MlpGateParams Q) { mlp_gemm<128, false, false, false, kGradXG>(P, nullptr, &G, &Q); }

int dm_mlp_smem_bytes(int bn) { return kMlpStages * (kMlpATile * 2 + 2 * bn * kMlpBK * 2) + 1024; }

template __global__ void dm_mlp_gemm_kernel<128, false>(MlpGemmParams);
template __global__ void dm_mlp_gemm_kernel<64, true>(MlpGemmParams);   // action sizes up to 64 (humanoid3d: 28, dog3d: 58)

}  // namespace dmk
