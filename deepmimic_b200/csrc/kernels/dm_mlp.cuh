// The host <-> kernel interface of the tensor-core network: the operand tile, the parameter structs the host fills and the kernels it
// launches (kernels/dm_mlp.cu, kernels/dm_learn.cu, kernels/dm_returns.cu; the launches are mlp_capi.cu's).  Every side includes this one
// definition: a struct that differed between the launching and the launched side would still compile and link, and the kernel would read its
// parameters at the wrong offsets.
#pragma once
#include <cuda_fp16.h>

#include <cstdint>

namespace dmk {

constexpr int kMlpBM = 128;          // rows per m tile (environments per CTA of the GEMMs)
constexpr int kMlpBK = 64;           // K elements per chunk (8 core matrices of 8 fp16)
constexpr int kMlpATile = kMlpBM * kMlpBK;   // halves per activation tile (16 KB): [k8][row group][row in group][8 halves]

// ---- the forward (kernels/dm_mlp.cu)
struct MlpPrepParams {
    const float* obs;          // [M x in_dim] fp32 observations
    const float* in_mean;      // normaliser mean / 1/std, in_dim entries
    const float* in_istd;
    float in_clip;
    int in_dim, M, NC;         // NC = padded K / 64
    __half* tiles;             // [m tiles][NC][kMlpATile]
    // gated actor only: the goal, normalised with its own statistics, fills the trunk columns [in_dim, in_dim + goal_dim) and, alone, the
    // gate trunk's 64-wide operand tile (written by the extra chunk blockIdx.y == NC)
    const float* goal;         // [M x goal_dim] fp32
    const float* g_mean;
    const float* g_istd;
    float g_clip;
    int goal_dim;
    __half* g_tiles;           // [m tiles][kMlpATile]
};
struct MlpGemmParams {
    const __half* a_tiles;     // [m tiles][K / 64][kMlpATile] fp16 activations in operand layout
    const __half* w_tiles;     // [n tiles][K / 64][hi | lo][BN x 64] in operand layout
    const float* bias;         // [N padded]
    __half* out_tiles;         // !LAST: [m tiles][N / 64][kMlpATile]
    float* actions;            // LAST: [M x out_dim] fp32
    const float* out_mean;     // LAST: action un-normalisation a * std + mean
    const float* out_std;
    const float* noise;        // LAST, optional: [M x out_dim] added in normalised action space (exploration), may be null
    int out_dim;
    int M, K, N;               // rows, padded K (multiple of 64), padded N (multiple of BN)
    // gated trunk layer only: two more K-chunks after the trunk's, both with this layer's gate-hidden chunk as A, against the gate's scale and
    // bias weights; the epilogue is relu(2 sigmoid(acc_s + bias_s) (acc + bias) + acc_b + bias_b)
    const __half* gate_tiles;  // A of the gate chunks: m tile t at gate_tiles + t * gate_stride
    const __half* ws_tiles;    // [n tiles][1][hi | lo][BN x 64]
    const __half* wb_tiles;
    const float* bias_s;       // [N padded]
    const float* bias_b;
    int gate_stride;           // halves
};
static_assert(sizeof(MlpGemmParams) == 128, "MlpGemmParams must stay at 128 bytes (see MlpStyleParams)");
// The discriminator head's outputs, a kernel parameter of its own: MlpGemmParams stays at 128 bytes (nvcc 12.9 compiles every GEMM
// instantiation differently once that struct grows past 128 bytes, even with the new fields unused).  Column 0 of the head is the logit
// d = acc + bias (no un-normalisation); per row r < M, style = max(0, 1 - 0.25 (1 - d)^2) and
// reward = (1 - task_lerp) style + task_lerp task_reward[r], or style without a task reward.
struct MlpStyleParams {
    const float* task_reward;  // [M] or null
    float* logit;              // [M] or null
    float* style;              // [M] or null
    float* reward;             // [M]
    float task_lerp;
};
// The backward GEMMs of the PPO learner (kernels/dm_learn.cu, mlp_capi.cu: dm_learn_step), also a parameter struct of their own; their modes
// GRAD_X, GRAD_W, GRAD_XA, GRAD_XG and SAVE are described in kernels/dm_mlp.cu
struct MlpGradParams {
    const __half* mask_tiles;  // GRAD_X: the layer's input activations, [m tiles][N / 64][kMlpATile] (GRAD_XA: or null, no mask)
    __half* dy_a;              // GRAD_X: dH in operand layout [m tiles][hi: N / 64, lo: N / 64][kMlpATile], or null
    __half* dy_b;              // GRAD_X: dH as B of the dW GEMM, [N / 128][row_chunks][hi | lo][128 x 64]
    float* partial;            // GRAD_W: [splits][N][M] (the parameter's [out x in] order)
    int row_chunks;            // minibatch rows / 64 (padded)
    int chunks_per_split;      // GRAD_W
};
// The gated layers' factors and gate operands (GRAD_XG, SAVE), a parameter struct of their own for the reason MlpStyleParams is
struct MlpGateParams {
    float* fa;                 // [M padded][N] fp32: 2 sigmoid(s)
    float* fb;                 // [M padded][N] fp32: 2 sigmoid(s) (1 - sigmoid(s)) z
    __half* st_a;              // GRAD_XG: A of the gate's dX GEMM, [m tiles][hi: st_nc, lo: st_nc][kMlpATile]; ds_l in chunks s_chunk + n / 64,
    int st_nc, s_chunk, t_chunk;   // dt_l in chunks t_chunk + n / 64
    __half* st_b;              // GRAD_XG: [2 N / 128][row_chunks][hi | lo][128 x 64], ds_l in n tiles [0, N / 128), dt_l in [N / 128, 2 N / 128)
};

// ---- the learner's steps (kernels/dm_learn.cu)
struct LearnPrepParams {
    const float* x;            // [samples x in_dim] fp32 window
    const int64_t* idx;        // [M] window sample of each minibatch row
    const float* mean;
    const float* istd;
    float clip;
    int in_dim, M, NC;         // NC = padded K / 64
    __half* tiles;             // [m tiles][NC][kMlpATile]
};
struct LearnTransposeParams {
    const __half* src[3];      // forward activations in operand layout [m tiles][src_nc][kMlpATile]
    __half* dst[3];            // transposed: [F / 128][row_chunks][kMlpATile], M = feature, K = minibatch row
    int src_nc[3];
    int ones[3];               // the feature that is 1 on every row (the layer's input size): its dW row is the bias gradient
    int F[3];                  // padded features (multiple of 128)
    int row_chunks;
};
struct LearnHeadParams {
    const float* out;          // [M x out_dim] the network's normalised output (mu, or the normalised value)
    const int64_t* idx;        // [M] window sample of each row
    int M, out_dim;
    __half* dy_a;              // [m tiles][hi | lo][kMlpATile]: A of the output layer's dX GEMM
    __half* dy_b;              // [1][row chunks][hi | lo][64 x 64]: B of the output layer's dW GEMM
    float* partials;           // [CTAs][3]
    // actor (PPOAgent._build_losses): normalised actions, old log-probabilities and advantages of the window, log sigma and the normalised
    // action bounds per action, the ratio clip; ratio: [M] per-row probability ratios, or null
    const float* actions;
    const float* old_logp;
    const float* adv;
    const float* logstd;
    const float* bound_min;
    const float* bound_max;
    float ratio_clip;
    float* ratio;
    // critic: the window's normalised, clipped targets
    const float* targets;
};
struct LearnLayerParams {
    float* w;                  // [out x in] fp32 (torch layout), updated in place
    float* b;                  // [out]
    float* acc_w;              // momentum accumulators, or null: re-tile only
    float* acc_b;
    const float* partial;      // [splits][Npad][F] dW partials; row in_dim holds db
    int splits, Npad, F;
    float inv_rows, lr, mom, wd;
    int in_dim, out_dim;
    __half* tiles;             // forward hi + lo tiles [Npad / BN][NC][2][BN x 64] (dm_mlp w[l])
    float* bias_pad;           // dm_mlp b[l]
    int NC, BN;
    __half* t_tiles;           // W^T hi + lo tiles of the dX GEMM [in tiles of 128][t_NC][2][128 x 64], or null
    int t_NC;
};
// the gated networks' goal (dm_learn_gated_step): [goal samples x goal_dim] fp32 window, normalised and clipped with its own statistics
struct LearnGoalParams {
    const float* goal;
    const float* g_mean;
    const float* g_istd;
    float g_clip;
    int goal_dim;
    __half* g_tiles;           // [m tiles][kMlpATile]: the normalised goal alone, the gate trunk's operand
};
struct LearnDiscHeadParams {
    const float* out;          // [2E] logits
    int rows, E;
    __half* dy_a;              // dY of the logit layer over all 2E rows, as LearnHeadParams::dy_a / dy_b
    __half* dy_b;
    __half* seed_a;            // dd / dd = 1 on the real expert rows (0 on their padding), over the E expert rows: A of the penalty's first dX
    __half* seed_b;            // GEMM, and B of its logit-weight dW GEMM
    float* partials;           // [2E / 128][3]: sum of (d -+ 1)^2, rows on the right side of 0, sum of d
};
struct LearnDiscLayerParams {
    LearnLayerParams L;        // as dm_learn_layer_kernel; t_tiles for every layer (layer 0's W0^T feeds the penalty's input-gradient GEMM)
    const float* pen;          // [pen_splits][L.Npad][pen_F] dW partials of 0.5 sum ||g||^2 (no bias term), or null: no penalty
    int pen_splits, pen_F;
    float gp_w;                // the penalty's weight
    float reg;                 // weight decay on top of L.wd for this layer's weights (the logit layer: logit_reg_weight)
    __half* p_tiles;           // layer 0, or null: W0's forward tiles with K padded to p_NC * 64 (B of the penalty's W0 e GEMM)
    int p_NC;
};
// one parameter pair's slice of a flat gradient buffer (dm_learn_grad, dm_learn_apply): w [out x in], b [out]; the apply pass reads scale * it
struct LearnGradParams {
    float* w;
    float* b;
    float scale;
};

// ---- kernels/dm_mlp.cu
__global__ void dm_mlp_prep_kernel(MlpPrepParams);
__global__ void dm_mlp_gated_prep_kernel(MlpPrepParams);
template <int BN, bool LAST>
__global__ void dm_mlp_gemm_kernel(MlpGemmParams);
__global__ void dm_mlp_gated_gemm_kernel(MlpGemmParams);
__global__ void dm_mlp_style_reward_kernel(MlpGemmParams, MlpStyleParams);
__global__ void dm_mlp_grad_x_kernel(MlpGemmParams, MlpGradParams);
template <int BN>
__global__ void dm_mlp_grad_w_kernel(MlpGemmParams, MlpGradParams);
__global__ void dm_mlp_grad_xa_kernel(MlpGemmParams, MlpGradParams);
__global__ void dm_mlp_gated_save_kernel(MlpGemmParams, MlpGateParams);
__global__ void dm_mlp_grad_xg_kernel(MlpGemmParams, MlpGradParams, MlpGateParams);
int dm_mlp_smem_bytes(int bn);   // dynamic shared memory of a GEMM launch with BN-column tiles
// ---- kernels/dm_returns.cu
__global__ void dm_td_lambda_kernel(const float*, const float*, const float*, const uint8_t*, const int32_t*, int, int, float, float, float, float, float*, float*);
// ---- kernels/dm_learn.cu
__global__ void dm_learn_prep_kernel(LearnPrepParams);
__global__ void dm_learn_gated_prep_kernel(LearnPrepParams, LearnGoalParams);
__global__ void dm_learn_transpose_kernel(LearnTransposeParams);
__global__ void dm_learn_actor_head_kernel(LearnHeadParams);
__global__ void dm_learn_critic_head_kernel(LearnHeadParams);
__global__ void dm_learn_stats_kernel(const float*, int, float, int, float*);
__global__ void dm_learn_layer_kernel(LearnLayerParams);
__global__ void dm_learn_norm_kernel(const float*, const float*, int, float*, float*, int);
__global__ void dm_learn_disc_head_kernel(LearnDiscHeadParams);
__global__ void dm_learn_disc_gp_kernel(const __half*, int, float*);
__global__ void dm_learn_disc_stats_kernel(const float*, int, const float*, int, float, float*);
__global__ void dm_learn_disc_layer_kernel(LearnDiscLayerParams);
__global__ void dm_learn_pack_kernel(LearnDiscLayerParams, LearnGradParams);
__global__ void dm_learn_apply_kernel(LearnDiscLayerParams, LearnGradParams);

}  // namespace dmk
