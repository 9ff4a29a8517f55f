// C ABI of the tensor-core policy network (include/deepmimic_b200.h, dm_mlp_*): host-side weight tiling + the launches of kernels/dm_mlp.cu: four for
// the plain actor (operand preparation, three GEMMs), six for the gated one (operand preparation, gate trunk, both gate hidden layers, two gated
// trunk layers, output layer), four for the AMP discriminator's style reward (operand preparation, two GEMMs, the logit head with the reward
// epilogue); the learner-side TD(lambda) return scan of a rollout window (kernels/dm_returns.cu, one launch); and the PPO learner's minibatch
// step (dm_learn_*: kernels/dm_learn.cu and the backward GEMMs of kernels/dm_mlp.cu, 15 launches; 32 for the gated networks,
// dm_learn_gated_step), the same step split around a flat gradient for data-parallel training (dm_learn_*grad, dm_learn_*apply), with the
// device-side re-tiling of plain and gated handles (dm_mlp_set_weights_device, dm_mlp_set_gated_weights_device).
// Every dm_learn_* step, grad, apply and set-weights entry is one call of `learn`, the checks, forward, backward and layer pass of its
// network family; every device buffer of a dm_mlp or dm_learn handle is allocated by `alloc` or `upload`, which record it for destroy.
// The parameter structs and kernel declarations are kernels/dm_mlp.cuh, shared with the kernels.
// Same library, same rules: no CPU fallback, errors through dm_last_error.
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <iterator>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/deepmimic_b200.h"
#include "kernels/dm_mlp.cuh"

extern "C" void dm_set_last_error(const char* msg);

// the clip of a normalised input before its fp16 operand: the caller's (<= 0: none), never past fp16's largest finite value, so an input
// the normaliser puts beyond +-65504 saturates there instead of reaching the GEMMs as inf (in range, the operand's bits do not change)
constexpr float kNoClip = 65504.f;
inline float operand_clip(float clip) { return clip > 0.f && clip < kNoClip ? clip : kNoClip; }

struct dm_mlp {
    int device = 0, in_dim = 0, h0 = 0, h1 = 0, out_dim = 0, max_rows = 0;
    int K0 = 0, N0 = 0, N1 = 0, N2 = 64;  // padded sizes: K0 = pad64(in), N0 = pad128(h0) = K1, N1 = pad128(h1) = K2, N2 = 64 (gated: K0 = pad64(in + goal), pad64(h))
    __half *w[3] = {nullptr, nullptr, nullptr}, *obs_t = nullptr, *act0 = nullptr, *act1 = nullptr;   // activations: operand tiles [m tiles][K / 64][128 x 64]
    float *b[3] = {nullptr, nullptr, nullptr}, *in_mean = nullptr, *in_istd = nullptr, *out_mean = nullptr, *out_std = nullptr;
    float in_clip = kNoClip;
    long long launches = 0;
    // gated actor (dm_mlp_create_gated) only: gate trunk (goal -> 128), both gate hidden layers as one 128 -> 128 GEMM (layer l in columns
    // [64 l, 64 l + 64)), per trunk layer the gate's scale and bias weights (64 -> h_l)
    bool gated = false;
    int goal_dim = 0, gate_common = 0, gate_hidden = 0;
    __half *wgc = nullptr, *wgh = nullptr, *wgs[2] = {nullptr, nullptr}, *wgb[2] = {nullptr, nullptr}, *goal_t = nullptr, *gc_t = nullptr, *gh_t = nullptr;
    float *bgc = nullptr, *bgh = nullptr, *bgs[2] = {nullptr, nullptr}, *bgb[2] = {nullptr, nullptr}, *g_mean = nullptr, *g_istd = nullptr;
    float g_clip = kNoClip;
    std::vector<void*> bufs;   // every device buffer the handle owns (alloc, upload), freed by dm_mlp_destroy
};

namespace {
int mlp_fail(const std::string& m) { dm_set_last_error(m.c_str()); std::fprintf(stderr, "[deepmimic_b200] %s\n", m.c_str()); return 1; }
// the outcome of the launches `fn` just enqueued: 0, or 1 with the launch error in dm_last_error
int launch_status(const char* fn) {
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : mlp_fail(std::string(fn) + ": " + cudaGetErrorString(e));
}
int pad_to(int v, int q) { return ((v + q - 1) / q) * q; }
// w: [K_in x N_out] row major (the reference's dense kernels: inputs x units).  Tiles: [n tile][k chunk][hi | lo][k8][row group][row][8 halves]
std::vector<__half> tile_weights(const float* w, int k_in, int n_out, int K, int N, int BN) {
    const int NC = K / 64, NT = N / BN;
    std::vector<__half> out(static_cast<size_t>(NT) * NC * 2 * BN * 64);
    for (int nt = 0; nt < NT; ++nt)
        for (int c = 0; c < NC; ++c) {
            __half* hi = &out[(static_cast<size_t>(nt) * NC + c) * 2 * BN * 64];
            __half* lo = hi + BN * 64;
            for (int k8 = 0; k8 < 8; ++k8)
                for (int rg = 0; rg < BN / 8; ++rg)
                    for (int r = 0; r < 8; ++r)
                        for (int e = 0; e < 8; ++e) {
                            const int n = nt * BN + rg * 8 + r, k = c * 64 + k8 * 8 + e;
                            const float v = (n < n_out && k < k_in) ? w[static_cast<size_t>(k) * n_out + n] : 0.f;
                            const __half h = __float2half_rn(v);
                            const size_t o = (static_cast<size_t>(k8) * (BN / 8) + rg) * 64 + r * 8 + e;
                            hi[o] = h; lo[o] = __float2half_rn(v - __half2float(h));
                        }
        }
    return out;
}
// a device buffer of `count` T (zeroed: cleared there) that handle h owns until its destroy function
template <class H, class T>
bool alloc(H* h, T** p, size_t count, bool zeroed = false) {
    if (cudaMalloc(p, count * sizeof(T)) != cudaSuccess) return false;
    h->bufs.push_back(*p);
    return !zeroed || cudaMemset(*p, 0, count * sizeof(T)) == cudaSuccess;
}
// a device buffer that handle h owns, holding a copy of src
template <class H, class T>
bool upload(H* h, T** dst, const std::vector<T>& src) {
    return alloc(h, dst, src.size()) && cudaMemcpy(*dst, src.data(), src.size() * sizeof(T), cudaMemcpyHostToDevice) == cudaSuccess;
}
std::vector<float> padded(const float* v, int n, int N, float fill = 0.f) { std::vector<float> o(N, fill); if (v) std::memcpy(o.data(), v, sizeof(float) * n); return o; }
std::vector<float> inverse_std(const float* std_dev, int n) { std::vector<float> o(n, 1.f); for (int i = 0; i < n; ++i) o[i] = std_dev ? 1.0f / std_dev[i] : 1.f; return o; }
// the create functions' device checks: a CUDA device is present, `device` can be selected and is an sm_90 part.  fn names the caller in error
// messages
bool device_ok(const std::string& fn, int device) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { mlp_fail(fn + ": no CUDA device (the policy network has no CPU fallback)"); return false; }
    if (cudaSetDevice(device) != cudaSuccess) { mlp_fail(fn + ": cudaSetDevice failed"); return false; }
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, device);
    if (prop.major != 9 || prop.minor != 0) { mlp_fail(fn + ": the wgmma kernels are built for sm_90a (found sm_" + std::to_string(prop.major) + std::to_string(prop.minor) + ")"); return false; }
    return true;
}
// the plain network's two hidden layers over the m tiles of `rows` rows prepared in obs_t (two launches); the caller sets the output layer's
// fields of the returned parameters and launches it
dmk::MlpGemmParams plain_hidden(const dm_mlp* m, int rows, cudaStream_t st) {
    const int mt = (rows + 127) / 128;
    dmk::MlpGemmParams P{};
    P.M = rows;
    // layer 0: 227 -> 1024 + ReLU
    P.a_tiles = m->obs_t; P.w_tiles = m->w[0]; P.bias = m->b[0]; P.out_tiles = m->act0; P.K = m->K0; P.N = m->N0;
    dmk::dm_mlp_gemm_kernel<128, false><<<dim3(mt, m->N0 / 128), 256, dmk::dm_mlp_smem_bytes(128), st>>>(P);
    // layer 1: 1024 -> 512 + ReLU
    P.a_tiles = m->act0; P.w_tiles = m->w[1]; P.bias = m->b[1]; P.out_tiles = m->act1; P.K = m->N0; P.N = m->N1;
    dmk::dm_mlp_gemm_kernel<128, false><<<dim3(mt, m->N1 / 128), 256, dmk::dm_mlp_smem_bytes(128), st>>>(P);
    // the output layer reads layer 1's tiles
    P.a_tiles = m->act1; P.w_tiles = m->w[2]; P.bias = m->b[2]; P.out_tiles = nullptr; P.K = m->N1; P.N = m->N2;
    return P;
}
// the gated network's gate trunk, both gate hidden layers and two gated trunk layers over the m tiles of `rows` rows prepared in obs_t and
// goal_t (four launches).  Given the learner's factor buffers (save[l] for trunk layer l) the trunk layers also save their factors
// (dm_mlp_gated_save_kernel); the caller sets the output layer's fields of the returned parameters and launches it
dmk::MlpGemmParams gated_hidden(const dm_mlp* m, int rows, const dmk::MlpGateParams* save, cudaStream_t st) {
    const int mt = (rows + 127) / 128;
    dmk::MlpGemmParams P{};
    P.M = rows;
    // gate trunk: goal -> 128 + ReLU
    P.a_tiles = m->goal_t; P.w_tiles = m->wgc; P.bias = m->bgc; P.out_tiles = m->gc_t; P.K = 64; P.N = 128;
    dmk::dm_mlp_gemm_kernel<128, false><<<dim3(mt, 1), 256, dmk::dm_mlp_smem_bytes(128), st>>>(P);
    // both gate hidden layers: 128 -> 2 x 64 + ReLU; K-chunk l of the output is layer l's gate in operand layout
    P.a_tiles = m->gc_t; P.w_tiles = m->wgh; P.bias = m->bgh; P.out_tiles = m->gh_t; P.K = 128; P.N = 128;
    dmk::dm_mlp_gemm_kernel<128, false><<<dim3(mt, 1), 256, dmk::dm_mlp_smem_bytes(128), st>>>(P);
    // gated trunk layers: 229 -> 1024, 1024 -> 512, each scaled and shifted by its gate
    auto gated = [&](int l) {
        if (save) dmk::dm_mlp_gated_save_kernel<<<dim3(mt, P.N / 64), 256, dmk::dm_mlp_smem_bytes(64), st>>>(P, save[l]);
        else dmk::dm_mlp_gated_gemm_kernel<<<dim3(mt, P.N / 64), 256, dmk::dm_mlp_smem_bytes(64), st>>>(P);
    };
    P.gate_stride = 2 * dmk::kMlpATile;
    P.a_tiles = m->obs_t; P.w_tiles = m->w[0]; P.bias = m->b[0]; P.out_tiles = m->act0; P.K = m->K0; P.N = m->N0;
    P.gate_tiles = m->gh_t; P.ws_tiles = m->wgs[0]; P.wb_tiles = m->wgb[0]; P.bias_s = m->bgs[0]; P.bias_b = m->bgb[0];
    gated(0);
    P.a_tiles = m->act0; P.w_tiles = m->w[1]; P.bias = m->b[1]; P.out_tiles = m->act1; P.K = m->N0; P.N = m->N1;
    P.gate_tiles = m->gh_t + dmk::kMlpATile; P.ws_tiles = m->wgs[1]; P.wb_tiles = m->wgb[1]; P.bias_s = m->bgs[1]; P.bias_b = m->bgb[1];
    gated(1);
    // the output layer reads layer 1's tiles
    P.a_tiles = m->act1; P.w_tiles = m->w[2]; P.bias = m->b[2]; P.out_tiles = nullptr; P.K = m->N1; P.N = m->N2;
    return P;
}
// the layer pass of kernels/dm_learn.cu for layer l of a plain handle: tiles of w[l] / b[l] from the fp32 [units x inputs] weights; the caller
// adds the optimiser's and the transposed tiles' fields
dmk::LearnLayerParams layer_params(dm_mlp* m, int l, const float* w, const float* b) {
    const int in[3] = {m->in_dim, m->h0, m->h1}, out[3] = {m->h0, m->h1, m->out_dim}, K[3] = {m->K0, m->N0, m->N1};
    dmk::LearnLayerParams L{};
    L.w = const_cast<float*>(w); L.b = const_cast<float*>(b); L.in_dim = in[l]; L.out_dim = out[l];
    L.tiles = m->w[l]; L.bias_pad = m->b[l]; L.NC = K[l] / 64; L.BN = l == 2 ? m->N2 : 128;
    return L;
}
void launch_layer(const dmk::LearnLayerParams& L, cudaStream_t st) {
    dmk::dm_learn_layer_kernel<<<dim3((L.in_dim + 1 + 255) / 256, L.out_dim), 256, 0, st>>>(L);
}
// parameter pair i of a gated handle, in dm_learn_gated_net's order W0, W1, W2, Wgc, Wgh_0, Wgh_1, Ws_0, Ws_1, Wt_0, Wt_1: the layer pass's fields
// for the forward tiles.  Both gate hidden layers share one 128-column matrix, layer l in columns [64 l, 64 l + GH): within a 128-wide tile,
// column 64 l + j sits 512 halves after column j, so the pass writes Wgh_l through shifted tile and bias pointers
dmk::LearnLayerParams gated_layer_params(dm_mlp* m, int i, const float* w, const float* b) {
    dmk::LearnLayerParams L{};
    L.w = const_cast<float*>(w); L.b = const_cast<float*>(b);
    const int GC = m->gate_common, GH = m->gate_hidden, l = i & 1;
    if (i < 3) {
        const int in[3] = {m->in_dim + m->goal_dim, m->h0, m->h1}, out[3] = {m->h0, m->h1, m->out_dim}, K[3] = {m->K0, m->N0, m->N1};
        L.in_dim = in[i]; L.out_dim = out[i]; L.tiles = m->w[i]; L.bias_pad = m->b[i]; L.NC = K[i] / 64; L.BN = 64;
    } else if (i == 3) {
        L.in_dim = m->goal_dim; L.out_dim = GC; L.tiles = m->wgc; L.bias_pad = m->bgc; L.NC = 1; L.BN = 128;
    } else if (i < 6) {
        L.in_dim = GC; L.out_dim = GH; L.tiles = m->wgh + 512 * l; L.bias_pad = m->bgh + 64 * l; L.NC = 2; L.BN = 128;
    } else {
        const bool scale = i < 8;
        L.in_dim = GH; L.out_dim = l ? m->h1 : m->h0; L.tiles = scale ? m->wgs[l] : m->wgb[l]; L.bias_pad = scale ? m->bgs[l] : m->bgb[l]; L.NC = 1; L.BN = 64;
    }
    return L;
}
// the optimiser step's fields of the layer pass of parameter pair i: its accumulators, the split count of its dW partials and the batch's 1 / rows,
// stepsize, momentum and weight decay
template <class Net, class Batch>
void optimiser_fields(dmk::LearnLayerParams& L, const Net* net, int i, const Batch* b, int splits) {
    L.acc_w = net->acc_w[i]; L.acc_b = net->acc_b[i]; L.splits = splits;
    L.inv_rows = 1.f / b->rows; L.lr = b->stepsize; L.mom = b->momentum; L.wd = b->weight_decay;
}
}  // namespace

// PPO learner workspace (include/deepmimic_b200.h: dm_learn_*).  Layer l = 0, 1, 2 has F[l] = pad128(inputs + 1) transposed-input features (the
// ones feature at index `inputs` makes row `inputs` of dW the bias gradient) and Nout[l] padded outputs (N0, N1, N2 of the handle).
struct dm_learn {
    dm_mlp* m = nullptr;
    int kind = 0;
    int max_rows = 0, F[3] = {0, 0, 0}, Nout[3] = {0, 0, 0}, max_splits[3] = {0, 0, 0};
    float* out = nullptr;                                    // [max_rows x out_dim] normalised network output
    __half *xt[3] = {nullptr, nullptr, nullptr};             // transposed saved activations: A of the dW GEMMs
    __half *dy_a[3] = {nullptr, nullptr, nullptr};           // dY of layers 1, 2 in operand layout, hi + lo chunks: A of the dX GEMMs (layer 0 needs none)
    __half *dy_b[3] = {nullptr, nullptr, nullptr};           // dY of every layer as hi + lo: B of the dW GEMMs
    __half *wt[3] = {nullptr, nullptr, nullptr};             // W1^T, W2^T as hi + lo: B of the dX GEMMs (kind 2: also W0^T)
    float *partial[3] = {nullptr, nullptr, nullptr}, *head_partials = nullptr;
    // kind 2, the discriminator's gradient penalty over the expert rows (at most E = pad128(max_rows / 2)), with the masks m_l = 1[a_l > 0]:
    //   u1 = m1 w2, u0 = m0 (W1^T u1), e = g = W0^T u0, q0 = m0 (W0 e), q1 = m1 (W1 q0);
    //   d(0.5 sum ||g||^2)/dW0 = sum u0 e^T, /dW1 = sum u1 q0^T, /dw2 = sum q1 (A of those dW GEMMs: e, q0, q1 transposed; B: u0, u1, the seed)
    int side_rows = 0, E = 0, Ng = 0, pen_F[3] = {0, 0, 0}, pen_max_splits[3] = {0, 0, 0};   // Ng = pad128(in_dim)
    __half *seed_a = nullptr, *seed_b = nullptr;             // dd/dd = 1 on the expert rows, A and B layouts of the logit layer's dY
    __half *u_a[2] = {nullptr, nullptr}, *u_b[2] = {nullptr, nullptr};   // u0, u1 as hi + lo A (next dX GEMM) and B (dW GEMM) operands
    __half *e_a = nullptr, *q_a[2] = {nullptr, nullptr};     // e, q0, q1 as hi + lo A operands
    __half *pt[3] = {nullptr, nullptr, nullptr};             // e, q0, q1 transposed: A of the penalty's dW GEMMs
    __half* w0p = nullptr;                                   // W0's forward tiles with K padded to Ng: B of the W0 e GEMM
    float *pen[3] = {nullptr, nullptr, nullptr}, *gp_partials = nullptr;
    // gated networks (dm_learn_create_gated): the trunk uses the fields of layers 0..2 above (dy_a[1] = dz_1); the handle pads the trunk to 128.
    // The gate's dW GEMMs j = 0..3: [Ws_0 | Wt_0] and [Ws_1 | Wt_1] (A = g_l transposed, B = [ds_l | dt_l]), [Wgh_0 | Wgh_1] (A = gc, B =
    // [dg_0 | dg_1]), Wgc (A = ng, B = dgc), each with gF[j] = pad128(inputs + 1) features and gN[j] outputs
    bool gated = false;
    int gF[4] = {0, 0, 0, 0}, gN[4] = {0, 0, 0, 0}, g_max_splits[4] = {0, 0, 0, 0};
    __half *gxt[4] = {nullptr, nullptr, nullptr, nullptr}, *gdy_b[4] = {nullptr, nullptr, nullptr, nullptr};
    float* gpartial[4] = {nullptr, nullptr, nullptr, nullptr};
    float *fa[2] = {nullptr, nullptr}, *fb[2] = {nullptr, nullptr};   // the gated layers' saved factors 2 sigma(s), 2 sigma(s) (1 - sigma(s)) z
    int KS = 0;                                              // chunks of [ds_0 | dt_0 | ds_1 | dt_1]: (2 N0 + 2 N1) / 64
    __half* st_a = nullptr;                                  // [ds_0 | dt_0 | ds_1 | dt_1] as hi + lo A of the dg GEMM
    __half* wst = nullptr;                                   // its B: Ws_l^T, Wt_l^T block-diagonal (layer l in columns [64 l, 64 l + GH))
    __half *dg_a = nullptr, *wght = nullptr;                 // [dg_0 | dg_1] as hi + lo A of the dgc GEMM, and its B: [Wgh_0 | Wgh_1]^T
    std::vector<void*> bufs;                                 // every device buffer of the workspace (alloc), freed by dm_learn_destroy
};

namespace {
// dm_mlp_create_gated with the trunk's widths padded to trunk_pad (64 for inference; the learner's own handle pads to 128, the width of the
// backward's tiles; the padding columns are zero and change no row's values).  fn names the caller in error messages
dm_mlp* create_gated(const char* fn, int device, const dm_mlp_gated_weights* g, int max_rows, int trunk_pad) {
    const std::string f(fn);
    if (!device_ok(f, device)) return nullptr;
    if (!g) { mlp_fail(f + ": null weights"); return nullptr; }
    if (g->in_dim <= 0 || g->goal_dim <= 0 || g->goal_dim > 64 || g->h0 <= 0 || g->h1 <= 0 || g->out_dim <= 0 || g->out_dim > 64 || max_rows <= 0) {
        mlp_fail(f + ": bad sizes (goal_dim must be <= 64, out_dim <= 64)"); return nullptr;
    }
    if (g->gate_common <= 0 || g->gate_common > 128 || g->gate_hidden <= 0 || g->gate_hidden > 64) {
        mlp_fail(f + ": unsupported gate sizes (gate_common must be <= 128, gate_hidden <= 64)"); return nullptr;
    }
    const float* need[] = {g->w0, g->b0, g->w1, g->b1, g->w2, g->b2, g->gc_w, g->gc_b, g->gh_w[0], g->gh_b[0], g->gh_w[1], g->gh_b[1],
                           g->gs_w[0], g->gs_b[0], g->gs_w[1], g->gs_b[1], g->gb_w[0], g->gb_b[0], g->gb_w[1], g->gb_b[1]};
    for (const float* p : need)
        if (!p) { mlp_fail(f + ": null weight pointer"); return nullptr; }
    dm_mlp* m = new dm_mlp();
    m->gated = true;
    m->device = device; m->in_dim = g->in_dim; m->goal_dim = g->goal_dim; m->gate_common = g->gate_common; m->gate_hidden = g->gate_hidden; m->h0 = g->h0; m->h1 = g->h1; m->out_dim = g->out_dim; m->max_rows = pad_to(max_rows, 128);
    const int trunk_in = g->in_dim + g->goal_dim, GC = g->gate_common, GH = g->gate_hidden;
    m->K0 = pad_to(trunk_in, 64); m->N0 = pad_to(g->h0, trunk_pad); m->N1 = pad_to(g->h1, trunk_pad);   // the gated layers run on 64-column tiles
    m->in_clip = operand_clip(g->s_clip);
    m->g_clip = operand_clip(g->g_clip);
    // both gate hidden layers side by side: layer l's GH units in columns [64 l, 64 l + GH), zero columns (relu(0) = 0) up to 64 l + 64
    std::vector<float> wgh(static_cast<size_t>(GC) * 128, 0.f), bgh(128, 0.f);
    for (int l = 0; l < 2; ++l) {
        for (int k = 0; k < GC; ++k)
            for (int n = 0; n < GH; ++n) wgh[static_cast<size_t>(k) * 128 + 64 * l + n] = g->gh_w[l][static_cast<size_t>(k) * GH + n];
        for (int n = 0; n < GH; ++n) bgh[64 * l + n] = g->gh_b[l][n];
    }
    const size_t R = m->max_rows;
    bool ok = upload(m, &m->w[0], tile_weights(g->w0, trunk_in, g->h0, m->K0, m->N0, 64)) && upload(m, &m->w[1], tile_weights(g->w1, g->h0, g->h1, m->N0, m->N1, 64)) &&
              upload(m, &m->w[2], tile_weights(g->w2, g->h1, g->out_dim, m->N1, m->N2, m->N2)) && upload(m, &m->b[0], padded(g->b0, g->h0, m->N0)) &&
              upload(m, &m->b[1], padded(g->b1, g->h1, m->N1)) && upload(m, &m->b[2], padded(g->b2, g->out_dim, m->N2)) &&
              upload(m, &m->wgc, tile_weights(g->gc_w, g->goal_dim, GC, 64, 128, 128)) && upload(m, &m->bgc, padded(g->gc_b, GC, 128)) &&
              upload(m, &m->wgh, tile_weights(wgh.data(), GC, 128, 128, 128, 128)) && upload(m, &m->bgh, bgh);
    const int hl[2] = {g->h0, g->h1}, Nl[2] = {m->N0, m->N1};
    for (int l = 0; l < 2 && ok; ++l)
        ok = upload(m, &m->wgs[l], tile_weights(g->gs_w[l], GH, hl[l], 64, Nl[l], 64)) && upload(m, &m->bgs[l], padded(g->gs_b[l], hl[l], Nl[l])) &&
             upload(m, &m->wgb[l], tile_weights(g->gb_w[l], GH, hl[l], 64, Nl[l], 64)) && upload(m, &m->bgb[l], padded(g->gb_b[l], hl[l], Nl[l]));
    // gh_t has one tile more than its rows need: the learner transposes layer 1's gate (chunk 1 of every m tile) as a two-chunk source, which
    // also reads the chunk after it (learn_gated_forward)
    ok = ok && upload(m, &m->in_mean, padded(g->s_mean, g->in_dim, g->in_dim)) && upload(m, &m->in_istd, inverse_std(g->s_std, g->in_dim)) &&
         upload(m, &m->g_mean, padded(g->g_mean, g->goal_dim, g->goal_dim)) && upload(m, &m->g_istd, inverse_std(g->g_std, g->goal_dim)) &&
         upload(m, &m->out_mean, padded(g->a_mean, g->out_dim, g->out_dim)) && upload(m, &m->out_std, padded(g->a_std, g->out_dim, g->out_dim, 1.f)) &&
         alloc(m, &m->obs_t, R * m->K0) && alloc(m, &m->goal_t, R * 64) && alloc(m, &m->gc_t, R * 128) && alloc(m, &m->gh_t, R * 128 + dmk::kMlpATile) &&
         alloc(m, &m->act0, R * m->N0) && alloc(m, &m->act1, R * m->N1);
    if (ok) {
        ok = cudaFuncSetAttribute(dmk::dm_mlp_gemm_kernel<128, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, dmk::dm_mlp_smem_bytes(128)) == cudaSuccess &&
             cudaFuncSetAttribute(dmk::dm_mlp_gated_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, dmk::dm_mlp_smem_bytes(64)) == cudaSuccess &&
             cudaFuncSetAttribute(dmk::dm_mlp_gemm_kernel<64, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, dmk::dm_mlp_smem_bytes(64)) == cudaSuccess;
    }
    if (!ok) { mlp_fail(f + ": " + cudaGetErrorString(cudaGetLastError())); dm_mlp_destroy(m); return nullptr; }
    return m;
}

// split-K of a dW GEMM: about two CTAs per SM of an H100 (132 SMs) over the (F / 128) x (N / BN) output tiles
void dw_split(int F, int N, int BN, int chunks, int* splits, int* cps) {
    const int tiles = (F / 128) * (N / BN);
    int s = std::max(1, std::min(chunks, (264 + tiles - 1) / tiles));
    *cps = (chunks + s - 1) / s;
    *splits = (chunks + *cps - 1) / *cps;
}
// the split count a dW GEMM's partials are sized for.  It is not monotonic in the row count (ceil(c / ceil(c / s))): the largest over every
// minibatch a step may take (an even chunk count up to max_chunks)
int dw_max_splits(int F, int N, int BN, int max_chunks) {
    int mx = 0;
    for (int c = 2; c <= max_chunks; c += 2) {
        int s = 0, cps = 0;
        dw_split(F, N, BN, c, &s, &cps);
        mx = std::max(mx, s);
    }
    return mx;
}
// a step's split-K plan of a dW GEMM over `chunks` row chunks, refused when it needs more partials than the workspace holds (max_splits)
int dw_plan(const char* fn, int F, int N, int BN, int chunks, int max_splits, int* splits, int* cps) {
    dw_split(F, N, BN, chunks, splits, cps);
    return *splits > max_splits ? mlp_fail(std::string(fn) + ": internal error: dW split count exceeds the workspace") : 0;
}
// dW = X^T dY over `chunks` row chunks, split into `splits` ranges of `cps` chunks: A = x_t (F transposed features), B = dy (N outputs on
// BN-column tiles), one fp32 partial product per split
void launch_dw(const __half* x_t, const __half* dy, float* partial, int F, int N, int BN, int chunks, int splits, int cps, cudaStream_t st) {
    dmk::MlpGemmParams W{};
    W.a_tiles = x_t; W.w_tiles = dy; W.M = F; W.N = N;
    const dmk::MlpGradParams GW{nullptr, nullptr, nullptr, partial, chunks, cps};
    if (BN == 64) dmk::dm_mlp_grad_w_kernel<64><<<dim3(F / 128, N / 64, splits), 256, dmk::dm_mlp_smem_bytes(64), st>>>(W, GW);
    else dmk::dm_mlp_grad_w_kernel<128><<<dim3(F / 128, N / 128, splits), 256, dmk::dm_mlp_smem_bytes(128), st>>>(W, GW);
}
// the column width of trunk layer i's dW GEMM: 128, the output layer's N2 = 64
int trunk_bn(const dm_learn* l, int i) { return i == 2 ? l->m->N2 : 128; }
// the workspace of the trunk's layers 0..2 (in[i] inputs), plain and gated: out, head_partials, F, Nout, xt, dy_a, dy_b, wt, partial (sized for
// the largest split count a step may take); and the backward kernels' shared-memory opt-in.  l->m and l->max_rows are set
bool trunk_workspace(dm_learn* l, const int* in) {
    const dm_mlp* m = l->m;
    const size_t R = l->max_rows;
    l->Nout[0] = m->N0; l->Nout[1] = m->N1; l->Nout[2] = m->N2;
    bool ok = alloc(l, &l->out, R * m->out_dim) && alloc(l, &l->head_partials, R / 128 * 3);
    for (int i = 0; i < 3 && ok; ++i) {
        l->F[i] = pad_to(in[i] + 1, 128);
        l->max_splits[i] = dw_max_splits(l->F[i], l->Nout[i], trunk_bn(l, i), l->max_rows / 64);
        ok = alloc(l, &l->xt[i], R * l->F[i]) && alloc(l, &l->dy_b[i], 2 * R * l->Nout[i]) &&
             alloc(l, &l->partial[i], static_cast<size_t>(l->max_splits[i]) * l->Nout[i] * l->F[i]);
        // W_i^T as B of the dX GEMM: K = Nout[i], N = Nout[i - 1] (zero padding written once)
        if (ok && i > 0) ok = alloc(l, &l->dy_a[i], 2 * R * l->Nout[i]) && alloc(l, &l->wt[i], 2 * static_cast<size_t>(l->Nout[i]) * l->Nout[i - 1], true);
    }
    return ok && cudaFuncSetAttribute(dmk::dm_mlp_grad_x_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, dmk::dm_mlp_smem_bytes(128)) == cudaSuccess &&
           cudaFuncSetAttribute(dmk::dm_mlp_grad_w_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, dmk::dm_mlp_smem_bytes(128)) == cudaSuccess &&
           cudaFuncSetAttribute(dmk::dm_mlp_grad_w_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, dmk::dm_mlp_smem_bytes(64)) == cudaSuccess;
}
}  // namespace

extern "C" {

dm_mlp* dm_mlp_create(int device, int in_dim, int h0, int h1, int out_dim, const float* w0, const float* b0, const float* w1, const float* b1, const float* w2, const float* b2,
                      const float* in_mean, const float* in_std, float in_clip, const float* out_mean, const float* out_std, int max_rows) {
    if (!device_ok("dm_mlp_create", device)) return nullptr;
    if (in_dim <= 0 || h0 <= 0 || h1 <= 0 || out_dim <= 0 || out_dim > 64 || max_rows <= 0) { mlp_fail("dm_mlp_create: bad sizes (out_dim must be <= 64)"); return nullptr; }
    dm_mlp* m = new dm_mlp();
    m->device = device; m->in_dim = in_dim; m->h0 = h0; m->h1 = h1; m->out_dim = out_dim; m->max_rows = pad_to(max_rows, 128);
    m->K0 = pad_to(in_dim, 64); m->N0 = pad_to(h0, 128); m->N1 = pad_to(h1, 128);
    m->in_clip = operand_clip(in_clip);
    const size_t R = m->max_rows;
    bool ok = upload(m, &m->w[0], tile_weights(w0, in_dim, h0, m->K0, m->N0, 128)) && upload(m, &m->w[1], tile_weights(w1, h0, h1, m->N0, m->N1, 128)) &&
              upload(m, &m->w[2], tile_weights(w2, h1, out_dim, m->N1, m->N2, m->N2)) && upload(m, &m->b[0], padded(b0, h0, m->N0)) && upload(m, &m->b[1], padded(b1, h1, m->N1)) &&
              upload(m, &m->b[2], padded(b2, out_dim, m->N2)) && upload(m, &m->in_mean, padded(in_mean, in_dim, in_dim)) && upload(m, &m->in_istd, inverse_std(in_std, in_dim)) &&
              upload(m, &m->out_mean, padded(out_mean, out_dim, out_dim)) && upload(m, &m->out_std, padded(out_std, out_dim, out_dim, 1.f)) &&
              alloc(m, &m->obs_t, R * m->K0) && alloc(m, &m->act0, R * m->N0) && alloc(m, &m->act1, R * m->N1);
    if (ok) {
        ok = cudaFuncSetAttribute(dmk::dm_mlp_gemm_kernel<128, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, dmk::dm_mlp_smem_bytes(128)) == cudaSuccess &&
             cudaFuncSetAttribute(dmk::dm_mlp_gemm_kernel<64, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, dmk::dm_mlp_smem_bytes(64)) == cudaSuccess;
    }
    if (ok && out_dim == 1)   // a one-unit head can be a discriminator (dm_mlp_forward_style_reward)
        ok = cudaFuncSetAttribute(dmk::dm_mlp_style_reward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, dmk::dm_mlp_smem_bytes(64)) == cudaSuccess;
    if (!ok) { mlp_fail(std::string("dm_mlp_create: ") + cudaGetErrorString(cudaGetLastError())); dm_mlp_destroy(m); return nullptr; }
    return m;
}

int dm_mlp_forward(dm_mlp* m, const float* d_obs, const float* d_noise, float* d_actions, int rows, void* stream) {
    if (!m) return mlp_fail("dm_mlp_forward: null handle");
    if (m->gated) return mlp_fail("dm_mlp_forward: the handle holds a gated actor (dm_mlp_create_gated); use dm_mlp_forward_gated");
    if (rows <= 0 || rows > m->max_rows) return mlp_fail("dm_mlp_forward: rows out of range");
    if (cudaSetDevice(m->device) != cudaSuccess) return mlp_fail("dm_mlp_forward: cudaSetDevice failed");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int mt = (rows + 127) / 128;
    // observations -> normalised fp16 operand tiles
    const dmk::MlpPrepParams Q{d_obs, m->in_mean, m->in_istd, m->in_clip, m->in_dim, rows, m->K0 / 64, m->obs_t};
    dmk::dm_mlp_prep_kernel<<<dim3(mt, m->K0 / 64), 128, 0, st>>>(Q);
    dmk::MlpGemmParams P = plain_hidden(m, rows, st);
    // layer 2: 512 -> actions, un-normalised
    P.actions = d_actions; P.out_mean = m->out_mean; P.out_std = m->out_std; P.noise = d_noise; P.out_dim = m->out_dim;
    dmk::dm_mlp_gemm_kernel<64, true><<<dim3(mt, 1), 256, dmk::dm_mlp_smem_bytes(64), st>>>(P);
    if (launch_status("dm_mlp_forward")) return 1;
    m->launches += 4;
    return 0;
}

dm_mlp* dm_mlp_create_gated(int device, const dm_mlp_gated_weights* g, int max_rows) {
    return create_gated("dm_mlp_create_gated", device, g, max_rows, 64);
}

int dm_mlp_forward_gated(dm_mlp* m, const float* d_obs, const float* d_goal, const float* d_noise, float* d_actions, int rows, void* stream) {
    if (!m) return mlp_fail("dm_mlp_forward_gated: null handle");
    if (!m->gated) return mlp_fail("dm_mlp_forward_gated: the handle holds a plain actor (dm_mlp_create); use dm_mlp_forward");
    if (!d_obs || !d_goal || !d_actions) return mlp_fail("dm_mlp_forward_gated: null observation, goal or action pointer");
    if (rows <= 0 || rows > m->max_rows) return mlp_fail("dm_mlp_forward_gated: rows out of range");
    if (cudaSetDevice(m->device) != cudaSuccess) return mlp_fail("dm_mlp_forward_gated: cudaSetDevice failed");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int mt = (rows + 127) / 128;
    // [state | goal] -> normalised fp16 trunk tiles; the normalised goal alone -> the gate trunk's tile (the extra chunk of the grid)
    dmk::MlpPrepParams Q{d_obs, m->in_mean, m->in_istd, m->in_clip, m->in_dim, rows, m->K0 / 64, m->obs_t, d_goal, m->g_mean, m->g_istd, m->g_clip, m->goal_dim, m->goal_t};
    dmk::dm_mlp_gated_prep_kernel<<<dim3(mt, m->K0 / 64 + 1), 128, 0, st>>>(Q);
    dmk::MlpGemmParams P = gated_hidden(m, rows, nullptr, st);
    // output layer: 512 -> actions, un-normalised
    P.actions = d_actions; P.out_mean = m->out_mean; P.out_std = m->out_std; P.noise = d_noise; P.out_dim = m->out_dim;
    dmk::dm_mlp_gemm_kernel<64, true><<<dim3(mt, 1), 256, dmk::dm_mlp_smem_bytes(64), st>>>(P);
    if (launch_status("dm_mlp_forward_gated")) return 1;
    m->launches += 6;
    return 0;
}

int dm_mlp_forward_style_reward(dm_mlp* m, const float* d_amp_obs, const float* d_task_reward, float task_lerp, float* d_logit, float* d_style, float* d_reward,
                                int rows, void* stream) {
    if (!m) return mlp_fail("dm_mlp_forward_style_reward: null handle");
    if (m->gated) return mlp_fail("dm_mlp_forward_style_reward: the handle holds a gated actor (dm_mlp_create_gated); a discriminator is a plain handle");
    if (m->out_dim != 1) return mlp_fail("dm_mlp_forward_style_reward: a discriminator has one output (out_dim " + std::to_string(m->out_dim) + ")");
    if (!(task_lerp >= 0.f && task_lerp <= 1.f)) return mlp_fail("dm_mlp_forward_style_reward: task_lerp must be in [0, 1]");
    if (rows <= 0 || rows > m->max_rows) return mlp_fail("dm_mlp_forward_style_reward: rows out of range");
    if (!d_amp_obs || !d_reward) return mlp_fail("dm_mlp_forward_style_reward: null AMP observation or reward pointer");
    if (cudaSetDevice(m->device) != cudaSuccess) return mlp_fail("dm_mlp_forward_style_reward: cudaSetDevice failed");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int mt = (rows + 127) / 128;
    const dmk::MlpPrepParams Q{d_amp_obs, m->in_mean, m->in_istd, m->in_clip, m->in_dim, rows, m->K0 / 64, m->obs_t};
    dmk::dm_mlp_prep_kernel<<<dim3(mt, m->K0 / 64), 128, 0, st>>>(Q);
    const dmk::MlpGemmParams P = plain_hidden(m, rows, st);
    // logit head: 512 -> 1, then the style reward and its blend with the task reward
    const dmk::MlpStyleParams S{d_task_reward, d_logit, d_style, d_reward, task_lerp};
    dmk::dm_mlp_style_reward_kernel<<<dim3(mt, 1), 256, dmk::dm_mlp_smem_bytes(64), st>>>(P, S);
    if (launch_status("dm_mlp_forward_style_reward")) return 1;
    m->launches += 4;
    return 0;
}

int dm_td_lambda_returns(const float* d_rewards, const float* d_values, const float* d_end_values, const uint8_t* d_done, const int32_t* d_terminate, int T, int N,
                         float discount, float td_lambda, float val_fail, float val_succ, float* d_returns, float* d_advantages, void* stream) {
    if (T <= 0 || N <= 0) return mlp_fail("dm_td_lambda_returns: T and N must be positive");
    if (!(discount >= 0.f && discount < 1.f)) return mlp_fail("dm_td_lambda_returns: discount must be in [0, 1)");
    if (!(td_lambda >= 0.f && td_lambda <= 1.f)) return mlp_fail("dm_td_lambda_returns: td_lambda must be in [0, 1]");
    if (!d_rewards || !d_values || !d_end_values || !d_done || !d_terminate || !d_returns || !d_advantages) return mlp_fail("dm_td_lambda_returns: null pointer");
    constexpr int kThreads = 64;   // N = 4096 environments -> 64 CTAs on 64 SMs: the scan is latency-bound, more SMs keep more loads in flight
    dmk::dm_td_lambda_kernel<<<(N + kThreads - 1) / kThreads, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        d_rewards, d_values, d_end_values, d_done, d_terminate, T, N, discount, td_lambda, val_fail, val_succ, d_returns, d_advantages);
    return launch_status("dm_td_lambda_returns");
}

int dm_mlp_set_weights_device(dm_mlp* m, const float* d_w0, const float* d_b0, const float* d_w1, const float* d_b1, const float* d_w2, const float* d_b2,
                              void* stream) {
    if (!m) return mlp_fail("dm_mlp_set_weights_device: null handle");
    if (m->gated) return mlp_fail("dm_mlp_set_weights_device: the handle holds a gated actor; only plain handles are re-tiled on the device");
    const float* p[6] = {d_w0, d_b0, d_w1, d_b1, d_w2, d_b2};
    for (const float* q : p)
        if (!q) return mlp_fail("dm_mlp_set_weights_device: null weight pointer");
    if (cudaSetDevice(m->device) != cudaSuccess) return mlp_fail("dm_mlp_set_weights_device: cudaSetDevice failed");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    for (int l = 0; l < 3; ++l) launch_layer(layer_params(m, l, p[2 * l], p[2 * l + 1]), st);
    return launch_status("dm_mlp_set_weights_device");
}

int dm_mlp_set_normalizers_device(dm_mlp* m, const float* d_in_mean, const float* d_in_std, const float* d_out_mean, const float* d_out_std, void* stream) {
    if (!m) return mlp_fail("dm_mlp_set_normalizers_device: null handle");
    if (m->gated) return mlp_fail("dm_mlp_set_normalizers_device: the handle holds a gated actor; only plain handles are refreshed on the device");
    if (!d_in_mean || !d_in_std || !d_out_mean || !d_out_std) return mlp_fail("dm_mlp_set_normalizers_device: null normaliser pointer");
    if (cudaSetDevice(m->device) != cudaSuccess) return mlp_fail("dm_mlp_set_normalizers_device: cudaSetDevice failed");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    dmk::dm_learn_norm_kernel<<<(m->in_dim + 255) / 256, 256, 0, st>>>(d_in_mean, d_in_std, m->in_dim, m->in_mean, m->in_istd, 1);
    dmk::dm_learn_norm_kernel<<<(m->out_dim + 255) / 256, 256, 0, st>>>(d_out_mean, d_out_std, m->out_dim, m->out_mean, m->out_std, 0);
    return launch_status("dm_mlp_set_normalizers_device");
}

dm_learn* dm_learn_create(int device, int kind, int in_dim, int h0, int h1, int out_dim, int max_rows) {
    if (kind != 0 && kind != 1 && kind != 2) { mlp_fail("dm_learn_create: kind must be 0 (actor), 1 (critic) or 2 (discriminator)"); return nullptr; }
    if (kind == 1 && out_dim != 1) { mlp_fail("dm_learn_create: a critic has one output"); return nullptr; }
    if (kind == 2 && out_dim != 1) { mlp_fail("dm_learn_create: a discriminator has one output"); return nullptr; }
    if (kind == 2 && max_rows == 1) { mlp_fail("dm_learn_create: a discriminator step needs max_rows >= 2 (one agent and one expert row)"); return nullptr; }
    if (in_dim <= 0 || h0 <= 0 || h1 <= 0 || out_dim <= 0 || out_dim > 64 || max_rows <= 0) { mlp_fail("dm_learn_create: bad sizes (out_dim must be <= 64)"); return nullptr; }
    // a discriminator's rows: the agent side in [0, E), the expert side in [E, 2 E), E = pad128(max_rows / 2)
    const int side = max_rows / 2, E = pad_to(side, 128), rows = kind == 2 ? 2 * E : max_rows;
    // zero weights and an identity output normaliser: dm_learn_set_weights loads the parameters, the output stays normalised
    std::vector<float> w0(static_cast<size_t>(in_dim) * h0), w1(static_cast<size_t>(h0) * h1), w2(static_cast<size_t>(h1) * out_dim), b0(h0), b1(h1), b2(out_dim);
    dm_mlp* m = dm_mlp_create(device, in_dim, h0, h1, out_dim, w0.data(), b0.data(), w1.data(), b1.data(), w2.data(), b2.data(), nullptr, nullptr, 0.f, nullptr, nullptr, rows);
    if (!m) return nullptr;   // dm_last_error is set
    dm_learn* l = new dm_learn();
    l->m = m; l->kind = kind; l->max_rows = m->max_rows;
    const int in[3] = {in_dim, h0, h1};
    bool ok = trunk_workspace(l, in);
    if (ok && kind == 2) {
        l->side_rows = side; l->E = E; l->Ng = pad_to(in_dim, 128);
        const int Ng = l->Ng, N0 = m->N0, N1 = m->N1;
        l->pen_F[0] = Ng; l->pen_F[1] = N0; l->pen_F[2] = N1;
        for (int i = 0; i < 3; ++i) l->pen_max_splits[i] = dw_max_splits(l->pen_F[i], l->Nout[i], trunk_bn(l, i), E / 64);
        const size_t e = E, tw = 2 * static_cast<size_t>(N0) * Ng;   // halves of W0^T / W0 as hi + lo tiles
        ok = alloc(l, &l->seed_a, 2 * e * 64) && alloc(l, &l->seed_b, 2 * e * 64) && alloc(l, &l->u_a[0], 2 * e * N0) && alloc(l, &l->u_b[0], 2 * e * N0) &&
             alloc(l, &l->u_a[1], 2 * e * N1) && alloc(l, &l->u_b[1], 2 * e * N1) && alloc(l, &l->e_a, 2 * e * Ng) && alloc(l, &l->q_a[0], 2 * e * N0) &&
             alloc(l, &l->q_a[1], 2 * e * N1) && alloc(l, &l->gp_partials, e / 128) && alloc(l, &l->wt[0], tw, true) && alloc(l, &l->w0p, tw, true);
        for (int i = 0; i < 3 && ok; ++i)
            ok = alloc(l, &l->pt[i], e * l->pen_F[i]) && alloc(l, &l->pen[i], static_cast<size_t>(l->pen_max_splits[i]) * l->Nout[i] * l->pen_F[i]);
        ok = ok && cudaFuncSetAttribute(dmk::dm_mlp_grad_xa_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, dmk::dm_mlp_smem_bytes(128)) == cudaSuccess;
    }
    if (!ok) { mlp_fail(std::string("dm_learn_create: ") + cudaGetErrorString(cudaGetLastError())); dm_learn_destroy(l); return nullptr; }
    return l;
}

}  // extern "C"

namespace {
// what a learner entry runs after its checks: the re-tiling alone (set-weights, no batch), the fused step (forward, backward, optimiser step
// and re-tiling), or one half of the split step: the mean gradient packed into a flat buffer (grad), or the optimiser step on scale times
// such a buffer (apply, no forward or backward)
enum class Pass { retile, step, pack, apply };
// the split counts of a step's dW GEMMs: the trunk's, the discriminator penalty's and the gate's.  A step's forward and backward fill them
// and its layer pass reads them; a re-tiling or an apply reads no dW partials and leaves them zero
struct Splits { int trunk[3] = {0, 0, 0}, pen[3] = {0, 0, 0}, gate[4] = {0, 0, 0, 0}; };
// the parameter and accumulator pointers of a plain (3 pairs) or gated (10 pairs) network
template <class Net>
int net_check(const char* fn, const Net* net) {
    if (!net) return mlp_fail(std::string(fn) + ": null parameters");
    for (size_t i = 0; i < std::size(net->w); ++i)
        if (!net->w[i] || !net->b[i] || !net->acc_w[i] || !net->acc_b[i]) return mlp_fail(std::string(fn) + ": null parameter or accumulator pointer");
    return 0;
}
// the checks of a PPO step's batch b; the gated step also passes gb (b = &gb->batch), whose goal pointers are checked with the states'
int batch_check(const char* fn, const dm_learn* l, const dm_learn_batch* b, const dm_learn_gated_batch* gb = nullptr) {
    const std::string f(fn);
    const bool actor = l->kind == 0;
    if (!b) return mlp_fail(f + ": null batch");
    if (b->rows <= 0 || b->rows > l->max_rows) return mlp_fail(f + ": rows out of range");
    if (!b->states || !b->idx || !b->in_mean || !b->in_istd || !b->stats || (gb && (!gb->goals || !gb->g_mean || !gb->g_istd)))
        return mlp_fail(f + (gb ? ": null state, goal, index, normaliser or statistics pointer" : ": null state, index, normaliser or statistics pointer"));
    if (actor && (!b->norm_actions || !b->old_logp || !b->adv || !b->logstd || !b->bound_min || !b->bound_max))
        return mlp_fail(f + ": null action, log-probability, advantage, log-std or bound pointer");
    if (!actor && !b->norm_targets) return mlp_fail(f + ": null target pointer");
    if (actor && !(b->ratio_clip > 0.f)) return mlp_fail(f + ": ratio_clip must be positive");
    if (!(b->stepsize >= 0.f) || !(b->momentum >= 0.f) || !(b->weight_decay >= 0.f)) return mlp_fail(f + ": stepsize, momentum and weight_decay must be >= 0");
    return 0;
}
int batch_check(const char* fn, const dm_learn* l, const dm_learn_gated_batch* gb) { return batch_check(fn, l, gb ? &gb->batch : nullptr, gb); }
int batch_check(const char* fn, const dm_learn* l, const dm_learn_disc_batch* b) {
    const std::string f(fn);
    if (!b) return mlp_fail(f + ": null batch");
    if (b->rows <= 0 || b->rows > l->side_rows) return mlp_fail(f + ": rows out of range (1 to max_rows / 2 per side)");
    if (!b->agent || !b->expert || !b->agent_idx || !b->expert_idx || !b->in_mean || !b->in_istd || !b->stats)
        return mlp_fail(f + ": null observation, index, normaliser or statistics pointer");
    if (!(b->stepsize >= 0.f) || !(b->momentum >= 0.f) || !(b->weight_decay >= 0.f) || !(b->logit_reg_weight >= 0.f) || !(b->grad_penalty_weight >= 0.f))
        return mlp_fail(f + ": stepsize, momentum, weight_decay, logit_reg_weight and grad_penalty_weight must be >= 0");
    return 0;
}
// a PPO step's loss head over the mt m tiles of l->out (dY of the output layer, the loss partials) and its statistics
void launch_ppo_head(const dm_learn* l, const dm_learn_batch* b, int mt, cudaStream_t st) {
    const bool actor = l->kind == 0;
    const dmk::LearnHeadParams H{l->out, b->idx, b->rows, l->m->out_dim, l->dy_a[2], l->dy_b[2], l->head_partials, b->norm_actions, b->old_logp, b->adv, b->logstd,
                                 b->bound_min, b->bound_max, b->ratio_clip, b->ratio, b->norm_targets};
    if (actor) dmk::dm_learn_actor_head_kernel<<<mt, 128, 0, st>>>(H);
    else dmk::dm_learn_critic_head_kernel<<<mt, 128, 0, st>>>(H);
    dmk::dm_learn_stats_kernel<<<1, 1, 0, st>>>(l->head_partials, mt, 1.f / b->rows, actor ? 1 : 0, b->stats);
}
// the pass of one parameter pair (disc: the discriminator's layer kernel for the re-tiling and the fused step); its slice of the flat gradient
// `grad` starts at *off (weights, then the bias), and *off moves past it
void launch_pass(Pass pass, const dmk::LearnDiscLayerParams& D, bool disc, float* grad, float scale, size_t* off, cudaStream_t st) {
    const dim3 grid((D.L.in_dim + 1 + 255) / 256, D.L.out_dim);
    const size_t nw = static_cast<size_t>(D.L.out_dim) * D.L.in_dim;
    const dmk::LearnGradParams G{grad ? grad + *off : nullptr, grad ? grad + *off + nw : nullptr, scale};
    *off += nw + D.L.out_dim;
    if (pass == Pass::pack) dmk::dm_learn_pack_kernel<<<grid, 256, 0, st>>>(D, G);
    else if (pass == Pass::apply) dmk::dm_learn_apply_kernel<<<grid, 256, 0, st>>>(D, G);
    else if (disc) dmk::dm_learn_disc_layer_kernel<<<grid, 256, 0, st>>>(D);
    else launch_layer(D.L, st);
}
// the layer passes of a plain workspace: the forward tiles of the learner's handle and the transposed tiles of the dX GEMMs (kind 2: also W0^T
// and W0's K-padded tiles for the penalty); with a batch `b` also the optimiser step on the dW partials (kind 2: with the penalty's partials
// and the logit regulariser), or the split step's pass: pack, apply on the flat gradient `grad`
template <class Batch>
void learn_layers(dm_learn* l, const dm_learn_net* net, const Batch* b, const Splits& s, Pass pass, float* grad, float scale, cudaStream_t st) {
    const bool disc = l->kind == 2;
    size_t off = 0;
    for (int i = 0; i < 3; ++i) {
        dmk::LearnDiscLayerParams D{};
        D.L = layer_params(l->m, i, net->w[i], net->b[i]);
        if (i > 0 || disc) { D.L.t_tiles = l->wt[i]; D.L.t_NC = l->Nout[i] / 64; }
        if (i == 0 && disc) { D.p_tiles = l->w0p; D.p_NC = l->Ng / 64; }
        if (b) {
            D.L.partial = l->partial[i]; D.L.Npad = l->Nout[i]; D.L.F = l->F[i];
            optimiser_fields(D.L, net, i, b, s.trunk[i]);
            if constexpr (std::is_same_v<Batch, dm_learn_disc_batch>) {
                D.pen = l->pen[i]; D.pen_splits = s.pen[i]; D.pen_F = l->pen_F[i]; D.gp_w = b->grad_penalty_weight; D.reg = i == 2 ? b->logit_reg_weight : 0.f;
            }
        }
        launch_pass(pass, D, disc, grad, scale, &off, st);
    }
}
// the forward over the mt m tiles prepared in the handle's obs_t (the output layer writes `rows` rows of l->out) and the transposition of the
// saved activations into the dW GEMMs' A operands
void learn_forward(dm_learn* l, int rows, int mt, cudaStream_t st) {
    dm_mlp* m = l->m;
    dmk::MlpGemmParams P = plain_hidden(m, rows, st);
    P.actions = l->out; P.out_mean = m->out_mean; P.out_std = m->out_std; P.noise = nullptr; P.out_dim = m->out_dim;
    dmk::dm_mlp_gemm_kernel<64, true><<<dim3(mt, 1), 256, dmk::dm_mlp_smem_bytes(64), st>>>(P);
    const int chunks = 2 * mt;
    dmk::LearnTransposeParams T{{m->obs_t, m->act0, m->act1}, {l->xt[0], l->xt[1], l->xt[2]}, {m->K0 / 64, m->N0 / 64, m->N1 / 64},
                                {m->in_dim, m->h0, m->h1}, {l->F[0], l->F[1], l->F[2]}, chunks};
    dmk::dm_learn_transpose_kernel<<<dim3(std::max(l->F[0], std::max(l->F[1], l->F[2])) / 128, chunks, 3), 256, 0, st>>>(T);
}
// backward of the dY a head wrote into dy_a[2] / dy_b[2], output layer first: dW_i = X_i^T dY_i (split K), dY_{i-1} = (dY_i W_i^T) * 1[X_i > 0]
void learn_backward(dm_learn* l, int rows, int mt, const int* splits, const int* cps, cudaStream_t st) {
    dm_mlp* m = l->m;
    const int chunks = 2 * mt;
    const __half* act[3] = {m->obs_t, m->act0, m->act1};
    for (int i = 2; i >= 0; --i) {
        launch_dw(l->xt[i], l->dy_b[i], l->partial[i], l->F[i], l->Nout[i], trunk_bn(l, i), chunks, splits[i], cps[i], st);
        if (i == 0) break;
        dmk::MlpGemmParams X{};
        X.a_tiles = l->dy_a[i]; X.w_tiles = l->wt[i]; X.M = rows; X.K = l->Nout[i]; X.N = l->Nout[i - 1];
        const dmk::MlpGradParams GX{act[i], i > 1 ? l->dy_a[i - 1] : nullptr, l->dy_b[i - 1], nullptr, chunks, 0};
        dmk::dm_mlp_grad_x_kernel<<<dim3(mt, l->Nout[i - 1] / 128), 256, dmk::dm_mlp_smem_bytes(128), st>>>(X, GX);
    }
}
// a PPO step up to its layer pass: the split-K plan of the three dW GEMMs (s.trunk), the forward, the loss head with its statistics and the
// backward
int forward_backward(const char* fn, dm_learn* l, const dm_learn_batch* b, Splits& s, cudaStream_t st) {
    dm_mlp* m = l->m;
    const int rows = b->rows, mt = (rows + 127) / 128, chunks = 2 * mt;
    // split-K of the three dW GEMMs for this row count (the workspace holds the largest over every row count, dm_learn_create)
    int cps[3];
    for (int i = 0; i < 3; ++i)
        if (dw_plan(fn, l->F[i], l->Nout[i], trunk_bn(l, i), chunks, l->max_splits[i], &s.trunk[i], &cps[i])) return 1;
    // forward: gathered rows -> the plain trunk -> the normalised output (identity output normaliser)
    dmk::LearnPrepParams Q{b->states, b->idx, b->in_mean, b->in_istd, operand_clip(b->in_clip), m->in_dim, rows, m->K0 / 64, m->obs_t};
    dmk::dm_learn_prep_kernel<<<dim3(mt, m->K0 / 64), 128, 0, st>>>(Q);
    learn_forward(l, rows, mt, st);
    // loss head: dY of the output layer, the loss partials, the statistics
    launch_ppo_head(l, b, mt, st);
    learn_backward(l, rows, mt, s.trunk, cps, st);
    return 0;
}
// a discriminator step up to its layer pass: the split-K plans of the dW GEMMs (s.trunk) and of the penalty's (s.pen), the forward over both
// sides, the least-squares head, the backward, the gradient penalty's GEMMs and the statistics
int forward_backward(const char* fn, dm_learn* l, const dm_learn_disc_batch* b, Splits& s, cudaStream_t st) {
    dm_mlp* m = l->m;
    // agent rows in m tiles [0, et), expert rows in [et, 2 et)
    const int rows = b->rows, E = pad_to(rows, 128), et = E / 128, mt = 2 * et, chunks = 2 * mt, echunks = 2 * et;
    int cps[3], pcps[3];
    for (int i = 0; i < 3; ++i)
        if (dw_plan(fn, l->F[i], l->Nout[i], trunk_bn(l, i), chunks, l->max_splits[i], &s.trunk[i], &cps[i]) ||
            dw_plan(fn, l->pen_F[i], l->Nout[i], trunk_bn(l, i), echunks, l->pen_max_splits[i], &s.pen[i], &pcps[i]))
            return 1;
    // forward over both sides: each gathered into its own m tiles
    const int NC0 = m->K0 / 64;
    dmk::LearnPrepParams Q{b->agent, b->agent_idx, b->in_mean, b->in_istd, operand_clip(b->in_clip), m->in_dim, rows, NC0, m->obs_t};
    dmk::dm_learn_prep_kernel<<<dim3(et, NC0), 128, 0, st>>>(Q);
    Q.x = b->expert; Q.idx = b->expert_idx; Q.tiles = m->obs_t + static_cast<size_t>(et) * NC0 * dmk::kMlpATile;
    dmk::dm_learn_prep_kernel<<<dim3(et, NC0), 128, 0, st>>>(Q);
    learn_forward(l, 2 * E, mt, st);
    // least-squares head: dY of the logit over both sides, the penalty's seed over the expert rows, the partials
    const dmk::LearnDiscHeadParams H{l->out, rows, E, l->dy_a[2], l->dy_b[2], l->seed_a, l->seed_b, l->head_partials};
    dmk::dm_learn_disc_head_kernel<<<mt, 128, 0, st>>>(H);
    learn_backward(l, 2 * E, mt, s.trunk, cps, st);
    // the gradient penalty on the expert tiles, with the forward's masks: u1 = m1 w2, u0 = m0 (W1^T u1) (hi + lo A and B operands) ...
    const size_t tile = dmk::kMlpATile;
    const __half* act0e = m->act0 + static_cast<size_t>(et) * (m->N0 / 64) * tile;
    const __half* act1e = m->act1 + static_cast<size_t>(et) * (m->N1 / 64) * tile;
    dmk::MlpGemmParams X{};
    X.M = E;
    X.a_tiles = l->seed_a; X.w_tiles = l->wt[2]; X.K = m->N2; X.N = m->N1;
    dmk::dm_mlp_grad_x_kernel<<<dim3(et, m->N1 / 128), 256, dmk::dm_mlp_smem_bytes(128), st>>>(X, dmk::MlpGradParams{act1e, l->u_a[1], l->u_b[1], nullptr, echunks, 0});
    X.a_tiles = l->u_a[1]; X.w_tiles = l->wt[1]; X.K = m->N1; X.N = m->N0;
    dmk::dm_mlp_grad_x_kernel<<<dim3(et, m->N0 / 128), 256, dmk::dm_mlp_smem_bytes(128), st>>>(X, dmk::MlpGradParams{act0e, l->u_a[0], l->u_b[0], nullptr, echunks, 0});
    // ... e = g = W0^T u0 (no mask), q0 = m0 (W0 e), q1 = m1 (W1 q0): hi + lo A operands only
    X.a_tiles = l->u_a[0]; X.w_tiles = l->wt[0]; X.K = m->N0; X.N = l->Ng;
    dmk::dm_mlp_grad_xa_kernel<<<dim3(et, l->Ng / 128), 256, dmk::dm_mlp_smem_bytes(128), st>>>(X, dmk::MlpGradParams{nullptr, l->e_a, nullptr, nullptr, echunks, 0});
    X.a_tiles = l->e_a; X.w_tiles = l->w0p; X.K = l->Ng; X.N = m->N0;
    dmk::dm_mlp_grad_xa_kernel<<<dim3(et, m->N0 / 128), 256, dmk::dm_mlp_smem_bytes(128), st>>>(X, dmk::MlpGradParams{act0e, l->q_a[0], nullptr, nullptr, echunks, 0});
    X.a_tiles = l->q_a[0]; X.w_tiles = m->w[1]; X.K = m->N0; X.N = m->N1;
    dmk::dm_mlp_grad_xa_kernel<<<dim3(et, m->N1 / 128), 256, dmk::dm_mlp_smem_bytes(128), st>>>(X, dmk::MlpGradParams{act1e, l->q_a[1], nullptr, nullptr, echunks, 0});
    dmk::dm_learn_disc_gp_kernel<<<et, 128, 0, st>>>(l->e_a, l->Ng / 64, l->gp_partials);
    // e, q0, q1 transposed (their hi chunks; no ones feature: the penalty has no bias gradient), then d(0.5 sum ||g||^2)/dW: sum u0 e^T,
    // sum u1 q0^T, sum q1 (B = the seed)
    const dmk::LearnTransposeParams T{{l->e_a, l->q_a[0], l->q_a[1]}, {l->pt[0], l->pt[1], l->pt[2]}, {2 * l->Ng / 64, 2 * m->N0 / 64, 2 * m->N1 / 64},
                                      {-1, -1, -1}, {l->pen_F[0], l->pen_F[1], l->pen_F[2]}, echunks};
    dmk::dm_learn_transpose_kernel<<<dim3(std::max(l->pen_F[0], std::max(l->pen_F[1], l->pen_F[2])) / 128, echunks, 3), 256, 0, st>>>(T);
    const __half* pen_b[3] = {l->u_b[0], l->u_b[1], l->seed_b};
    for (int i = 0; i < 3; ++i) launch_dw(l->pt[i], pen_b[i], l->pen[i], l->pen_F[i], l->Nout[i], trunk_bn(l, i), echunks, s.pen[i], pcps[i], st);
    dmk::dm_learn_disc_stats_kernel<<<1, 1, 0, st>>>(l->head_partials, mt, l->gp_partials, et, 1.f / rows, b->stats);
    return 0;
}
}  // namespace

extern "C" {

long long dm_learn_grad_size(const dm_learn* l) {
    if (!l) { mlp_fail("dm_learn_grad_size: null handle"); return -1; }
    long long n = 0;
    for (int i = 0; i < (l->gated ? 10 : 3); ++i) {
        const dmk::LearnLayerParams L = l->gated ? gated_layer_params(l->m, i, nullptr, nullptr) : layer_params(l->m, i, nullptr, nullptr);
        n += static_cast<long long>(L.out_dim) * (L.in_dim + 1);
    }
    return n;
}

dm_learn* dm_learn_create_gated(int device, int kind, int in_dim, int goal_dim, int h0, int h1, int out_dim, int gate_common, int gate_hidden, int max_rows) {
    if (kind != 0 && kind != 1) { mlp_fail("dm_learn_create_gated: kind must be 0 (actor) or 1 (critic)"); return nullptr; }
    if (kind == 1 && out_dim != 1) { mlp_fail("dm_learn_create_gated: a critic has one output"); return nullptr; }
    if (in_dim <= 0 || goal_dim <= 0 || goal_dim > 64 || h0 <= 0 || h1 <= 0 || out_dim <= 0 || out_dim > 64 || max_rows <= 0) {
        mlp_fail("dm_learn_create_gated: bad sizes (goal_dim must be <= 64, out_dim <= 64)"); return nullptr;
    }
    if (gate_common <= 0 || gate_common > 128 || gate_hidden <= 0 || gate_hidden > 64) {
        mlp_fail("dm_learn_create_gated: unsupported gate sizes (gate_common must be <= 128, gate_hidden <= 64)"); return nullptr;
    }
    // zero weights and identity normalisers (dm_learn_set_gated_weights loads the parameters, the output stays normalised); the trunk padded to
    // 128 columns, the width of the backward's tiles
    const int GC = gate_common, GH = gate_hidden, trunk_in = in_dim + goal_dim;
    std::vector<float> w0(static_cast<size_t>(trunk_in) * h0), w1(static_cast<size_t>(h0) * h1), w2(static_cast<size_t>(h1) * out_dim), b0(h0), b1(h1), b2(out_dim),
        gcw(static_cast<size_t>(goal_dim) * GC), gcb(GC), ghw(static_cast<size_t>(GC) * GH), ghb(GH), gw0(static_cast<size_t>(GH) * h0), gw1(static_cast<size_t>(GH) * h1);
    dm_mlp_gated_weights g{};
    g.in_dim = in_dim; g.goal_dim = goal_dim; g.h0 = h0; g.h1 = h1; g.out_dim = out_dim; g.gate_common = GC; g.gate_hidden = GH;
    g.w0 = w0.data(); g.b0 = b0.data(); g.w1 = w1.data(); g.b1 = b1.data(); g.w2 = w2.data(); g.b2 = b2.data(); g.gc_w = gcw.data(); g.gc_b = gcb.data();
    for (int i = 0; i < 2; ++i) {
        g.gh_w[i] = ghw.data(); g.gh_b[i] = ghb.data();
        g.gs_w[i] = g.gb_w[i] = i ? gw1.data() : gw0.data(); g.gs_b[i] = g.gb_b[i] = i ? b1.data() : b0.data();
    }
    dm_mlp* m = create_gated("dm_learn_create_gated", device, &g, max_rows, 128);
    if (!m) return nullptr;   // dm_last_error is set
    dm_learn* l = new dm_learn();
    l->m = m; l->gated = true; l->kind = kind; l->max_rows = m->max_rows;
    const int N0 = m->N0, N1 = m->N1, in[3] = {trunk_in, h0, h1};
    const int gF[4] = {128, 128, pad_to(GC + 1, 128), 128}, gN[4] = {2 * N0, 2 * N1, 128, 128};
    const size_t R = m->max_rows;
    l->KS = (2 * N0 + 2 * N1) / 64;
    bool ok = trunk_workspace(l, in);
    for (int j = 0; j < 4 && ok; ++j) {
        l->gF[j] = gF[j]; l->gN[j] = gN[j]; l->g_max_splits[j] = dw_max_splits(gF[j], gN[j], 128, m->max_rows / 64);
        ok = alloc(l, &l->gxt[j], R * gF[j]) && alloc(l, &l->gdy_b[j], 2 * R * gN[j]) && alloc(l, &l->gpartial[j], static_cast<size_t>(l->g_max_splits[j]) * gN[j] * gF[j]);
    }
    for (int i = 0; i < 2 && ok; ++i) ok = alloc(l, &l->fa[i], R * (i ? N1 : N0)) && alloc(l, &l->fb[i], R * (i ? N1 : N0));
    // the block-diagonal and transposed B operands keep their zero blocks and padding from here on (the layer passes write the weights only)
    ok = ok && alloc(l, &l->st_a, 2 * R * l->KS * 64) && alloc(l, &l->wst, 2 * static_cast<size_t>(l->KS) * 64 * 128, true) && alloc(l, &l->dg_a, 2 * R * 128) &&
         alloc(l, &l->wght, 2 * 128 * 128, true);
    if (ok) {
        ok = cudaFuncSetAttribute(dmk::dm_mlp_gated_save_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, dmk::dm_mlp_smem_bytes(64)) == cudaSuccess &&
             cudaFuncSetAttribute(dmk::dm_mlp_grad_xg_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, dmk::dm_mlp_smem_bytes(128)) == cudaSuccess;
    }
    if (!ok) { mlp_fail(std::string("dm_learn_create_gated: ") + cudaGetErrorString(cudaGetLastError())); dm_learn_destroy(l); return nullptr; }
    return l;
}

}  // extern "C"

namespace {
// chunk offsets of ds_l and dt_l in [ds_0 | dt_0 | ds_1 | dt_1]
int s_chunk(const dm_learn* l, int layer) { return layer ? 2 * l->m->N0 / 64 : 0; }
int t_chunk(const dm_learn* l, int layer) { return s_chunk(l, layer) + (layer ? l->m->N1 : l->m->N0) / 64; }
// the ten layer passes of a gated workspace: the forward tiles, and the B operands of the dX GEMMs (W1^T, W2^T, the block-diagonal
// [Ws_l^T, Wt_l^T], [Wgh_0 | Wgh_1]^T); with a batch `gb` also the optimiser step on the dW partials (split counts: sp.trunk for the trunk,
// sp.gate for the gate's GEMMs; or the split step's pass, as for a plain workspace)
void learn_layers(dm_learn* l, const dm_learn_gated_net* net, const dm_learn_gated_batch* gb, const Splits& sp, Pass pass, float* grad, float scale,
                  cudaStream_t st) {
    dm_mlp* m = l->m;
    const dm_learn_batch* b = gb ? &gb->batch : nullptr;
    const size_t tt = 2 * 128 * 64;   // halves of a hi + lo 128 x 64 B tile
    size_t off = 0;
    for (int i = 0; i < 10; ++i) {
        dmk::LearnDiscLayerParams D{};
        dmk::LearnLayerParams& L = D.L;
        L = gated_layer_params(m, i, net->w[i], net->b[i]);
        const int lay = i & 1;
        int s = 0;
        if (i < 3) {
            if (i > 0) { L.t_tiles = l->wt[i]; L.t_NC = l->Nout[i] / 64; }
            L.partial = l->partial[i]; L.Npad = l->Nout[i]; L.F = l->F[i]; s = sp.trunk[i];
        } else if (i == 3) {
            L.partial = l->gpartial[3]; L.Npad = 128; L.F = l->gF[3]; s = sp.gate[3];
        } else if (i < 6) {
            L.t_tiles = l->wght + lay * tt; L.t_NC = 2;
            L.partial = l->gpartial[2] + static_cast<size_t>(64 * lay) * l->gF[2]; L.Npad = 128; L.F = l->gF[2]; s = sp.gate[2];
        } else {
            const bool gate_scale = i < 8;
            const int N = lay ? m->N1 : m->N0;
            L.t_tiles = l->wst + static_cast<size_t>(gate_scale ? s_chunk(l, lay) : t_chunk(l, lay)) * tt + 512 * lay; L.t_NC = l->KS;
            L.partial = l->gpartial[lay] + (gate_scale ? 0 : static_cast<size_t>(N) * l->gF[lay]); L.Npad = 2 * N; L.F = l->gF[lay]; s = sp.gate[lay];
        }
        if (b) optimiser_fields(L, net, i, b, s);
        launch_pass(pass, D, false, grad, scale, &off, st);
    }
}
// the gated forward over the mt m tiles prepared in obs_t / goal_t (dm_mlp_forward_gated, with the gated layers saving their factors) and the
// transposition of the saved activations into the dW GEMMs' A operands
void learn_gated_forward(dm_learn* l, int rows, int mt, cudaStream_t st) {
    dm_mlp* m = l->m;
    const dmk::MlpGateParams save[2] = {{l->fa[0], l->fb[0], nullptr, 0, 0, 0, nullptr}, {l->fa[1], l->fb[1], nullptr, 0, 0, 0, nullptr}};
    dmk::MlpGemmParams P = gated_hidden(m, rows, save, st);
    P.actions = l->out; P.out_mean = m->out_mean; P.out_std = m->out_std; P.noise = nullptr; P.out_dim = m->out_dim;
    dmk::dm_mlp_gemm_kernel<64, true><<<dim3(mt, 1), 256, dmk::dm_mlp_smem_bytes(64), st>>>(P);
    // [ns | ng], h_0, h_1; then ng, gc, g_0 (chunk 0 of gh_t) and g_1 (chunk 1: a two-chunk source whose second chunk is never used, hence
    // gh_t's spare tile), each with its ones feature
    const int chunks = 2 * mt;
    const dmk::LearnTransposeParams T{{m->obs_t, m->act0, m->act1}, {l->xt[0], l->xt[1], l->xt[2]}, {m->K0 / 64, m->N0 / 64, m->N1 / 64},
                                      {m->in_dim + m->goal_dim, m->h0, m->h1}, {l->F[0], l->F[1], l->F[2]}, chunks};
    dmk::dm_learn_transpose_kernel<<<dim3(std::max(l->F[0], std::max(l->F[1], l->F[2])) / 128, chunks, 3), 256, 0, st>>>(T);
    const dmk::LearnTransposeParams G{{m->goal_t, m->gc_t, m->gh_t}, {l->gxt[3], l->gxt[2], l->gxt[0]}, {1, 2, 2}, {m->goal_dim, m->gate_common, m->gate_hidden},
                                      {l->gF[3], l->gF[2], l->gF[0]}, chunks};
    dmk::dm_learn_transpose_kernel<<<dim3(l->gF[2] / 128, chunks, 3), 256, 0, st>>>(G);
    const dmk::LearnTransposeParams G1{{m->gh_t + dmk::kMlpATile, nullptr, nullptr}, {l->gxt[1], nullptr, nullptr}, {2, 0, 0}, {m->gate_hidden, 0, 0}, {l->gF[1], 0, 0}, chunks};
    dmk::dm_learn_transpose_kernel<<<dim3(1, chunks, 1), 256, 0, st>>>(G1);
}
// the gated backward of the dY a head wrote into dy_a[2] / dy_b[2] (DESIGN.md section 8): dX GEMMs output -> h_1 -> h_0 with the gated
// epilogue (dz, ds, dt), the gate's dg and dgc GEMMs, and the seven split-K dW GEMMs
void learn_gated_backward(dm_learn* l, int mt, const int* splits, const int* cps, const int* gsplits, const int* gcps, cudaStream_t st) {
    dm_mlp* m = l->m;
    const int chunks = 2 * mt, N0 = m->N0, N1 = m->N1;
    launch_dw(l->xt[2], l->dy_b[2], l->partial[2], l->F[2], m->N2, m->N2, chunks, splits[2], cps[2], st);
    dmk::MlpGemmParams X{};
    X.a_tiles = l->dy_a[2]; X.w_tiles = l->wt[2]; X.K = m->N2; X.N = N1;
    dmk::dm_mlp_grad_xg_kernel<<<dim3(mt, N1 / 128), 256, dmk::dm_mlp_smem_bytes(128), st>>>(
        X, dmk::MlpGradParams{m->act1, l->dy_a[1], l->dy_b[1], nullptr, chunks, 0}, dmk::MlpGateParams{l->fa[1], l->fb[1], l->st_a, l->KS, s_chunk(l, 1), t_chunk(l, 1), l->gdy_b[1]});
    launch_dw(l->xt[1], l->dy_b[1], l->partial[1], l->F[1], N1, 128, chunks, splits[1], cps[1], st);
    launch_dw(l->gxt[1], l->gdy_b[1], l->gpartial[1], l->gF[1], l->gN[1], 128, chunks, gsplits[1], gcps[1], st);
    X.a_tiles = l->dy_a[1]; X.w_tiles = l->wt[1]; X.K = N1; X.N = N0;
    dmk::dm_mlp_grad_xg_kernel<<<dim3(mt, N0 / 128), 256, dmk::dm_mlp_smem_bytes(128), st>>>(
        X, dmk::MlpGradParams{m->act0, nullptr, l->dy_b[0], nullptr, chunks, 0}, dmk::MlpGateParams{l->fa[0], l->fb[0], l->st_a, l->KS, s_chunk(l, 0), t_chunk(l, 0), l->gdy_b[0]});
    launch_dw(l->xt[0], l->dy_b[0], l->partial[0], l->F[0], N0, 128, chunks, splits[0], cps[0], st);
    launch_dw(l->gxt[0], l->gdy_b[0], l->gpartial[0], l->gF[0], l->gN[0], 128, chunks, gsplits[0], gcps[0], st);
    // [dg_0 | dg_1] = ([ds_0 | dt_0 | ds_1 | dt_1] x block-diagonal [Ws_l^T; Wt_l^T]) * 1[g > 0], in gh_t's layout; dgc = ([dg_0 | dg_1] Wgh) * 1[gc > 0]
    X.a_tiles = l->st_a; X.w_tiles = l->wst; X.K = l->KS * 64; X.N = 128;
    dmk::dm_mlp_grad_x_kernel<<<dim3(mt, 1), 256, dmk::dm_mlp_smem_bytes(128), st>>>(X, dmk::MlpGradParams{m->gh_t, l->dg_a, l->gdy_b[2], nullptr, chunks, 0});
    launch_dw(l->gxt[2], l->gdy_b[2], l->gpartial[2], l->gF[2], 128, 128, chunks, gsplits[2], gcps[2], st);
    X.a_tiles = l->dg_a; X.w_tiles = l->wght; X.K = 128; X.N = 128;
    dmk::dm_mlp_grad_x_kernel<<<dim3(mt, 1), 256, dmk::dm_mlp_smem_bytes(128), st>>>(X, dmk::MlpGradParams{m->gc_t, nullptr, l->gdy_b[3], nullptr, chunks, 0});
    launch_dw(l->gxt[3], l->gdy_b[3], l->gpartial[3], l->gF[3], 128, 128, chunks, gsplits[3], gcps[3], st);
}
// a gated PPO step up to its layer passes: the split-K plans of the trunk's (s.trunk) and the gate's (s.gate) dW GEMMs, the forward, the
// loss head with its statistics and the gated backward
int forward_backward(const char* fn, dm_learn* l, const dm_learn_gated_batch* gb, Splits& s, cudaStream_t st) {
    dm_mlp* m = l->m;
    const dm_learn_batch* b = &gb->batch;
    const int rows = b->rows, mt = (rows + 127) / 128, chunks = 2 * mt;
    int cps[3], gcps[4];
    for (int i = 0; i < 3; ++i)
        if (dw_plan(fn, l->F[i], l->Nout[i], trunk_bn(l, i), chunks, l->max_splits[i], &s.trunk[i], &cps[i])) return 1;
    for (int j = 0; j < 4; ++j)
        if (dw_plan(fn, l->gF[j], l->gN[j], 128, chunks, l->g_max_splits[j], &s.gate[j], &gcps[j])) return 1;
    // forward: gathered [state | goal] rows and goals -> the gated network -> the normalised output (identity output normaliser)
    const dmk::LearnPrepParams Q{b->states, b->idx, b->in_mean, b->in_istd, operand_clip(b->in_clip), m->in_dim, rows, m->K0 / 64, m->obs_t};
    const dmk::LearnGoalParams Qg{gb->goals, gb->g_mean, gb->g_istd, operand_clip(gb->g_clip), m->goal_dim, m->goal_t};
    dmk::dm_learn_gated_prep_kernel<<<dim3(mt, m->K0 / 64 + 1), 128, 0, st>>>(Q, Qg);
    learn_gated_forward(l, rows, mt, st);
    // the loss heads act on the output only: the plain step's
    launch_ppo_head(l, b, mt, st);
    learn_gated_backward(l, mt, s.trunk, cps, s.gate, gcps, st);
    return 0;
}
// the workspace check of a learner entry: a gated entry needs a gated workspace, a plain one a plain workspace; beyond the re-tiling, the
// discriminator's entries need kind 2 and the PPO entries kind 0 or 1
int family_check(const char* fn, const dm_learn* l, bool gated, bool disc, Pass pass) {
    const std::string f(fn);
    if (!l) return mlp_fail(f + ": null handle");
    if (gated && !l->gated) return mlp_fail(f + ": the workspace holds a plain network (dm_learn_create)");
    if (!gated && l->gated) return mlp_fail(f + ": the workspace holds a gated network (dm_learn_create_gated)");
    if (pass == Pass::retile) return 0;
    if (disc && l->kind != 2) return mlp_fail(f + ": the workspace is a PPO actor's or critic's (kind 0 or 1); the discriminator's entries need kind 2");
    if (!disc && l->kind == 2) return mlp_fail(f + ": the workspace is a discriminator's (kind 2)");
    return 0;
}
// the checks of an apply: the optimiser fields it reads (a gated batch: those of its PPO batch), the flat gradient and its scale
template <class Batch>
int apply_check(const char* fn, const Batch* b, const float* d_grad, float scale) {
    if constexpr (std::is_same_v<Batch, dm_learn_gated_batch>) {
        return apply_check(fn, b ? &b->batch : nullptr, d_grad, scale);
    } else {
        const std::string f(fn);
        if (!b) return mlp_fail(f + ": null batch");
        if (!d_grad) return mlp_fail(f + ": null gradient pointer");
        if (!std::isfinite(scale)) return mlp_fail(f + ": scale must be finite");
        float reg = 0.f;
        if constexpr (std::is_same_v<Batch, dm_learn_disc_batch>) reg = b->logit_reg_weight;
        if (!(b->stepsize >= 0.f) || !(b->momentum >= 0.f) || !(b->weight_decay >= 0.f) || !(reg >= 0.f))
            return mlp_fail(f + ": stepsize, momentum, weight_decay (and logit_reg_weight) must be >= 0");
        return 0;
    }
}
// the dm_learn_* entry fn: the workspace check, the checks of the net and of the batch (an apply: apply_check), device and stream, the
// forward and backward of a step or grad (they fill the split counts), the layer pass and the launch status.  Net and Batch name the
// family: dm_learn_net with dm_learn_batch (the PPO networks; for set-weights, every plain workspace) or dm_learn_disc_batch, and
// dm_learn_gated_net with dm_learn_gated_batch.  b is null for the re-tiling
template <class Batch, class Net>
int learn(const char* fn, Pass pass, dm_learn* l, const Net* net, const Batch* b, float* grad, float scale, void* stream) {
    constexpr bool gated = std::is_same_v<Net, dm_learn_gated_net>, disc = std::is_same_v<Batch, dm_learn_disc_batch>;
    const bool steps = pass == Pass::step || pass == Pass::pack;   // a forward and backward before the layer pass
    if (family_check(fn, l, gated, disc, pass) || net_check(fn, net)) return 1;
    if (steps && batch_check(fn, l, b)) return 1;
    if (pass == Pass::apply && apply_check(fn, b, grad, scale)) return 1;
    if (pass == Pass::pack && !grad) return mlp_fail(std::string(fn) + ": null gradient pointer");
    if (cudaSetDevice(l->m->device) != cudaSuccess) return mlp_fail(std::string(fn) + ": cudaSetDevice failed");
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    Splits s;
    if (steps && forward_backward(fn, l, b, s, st)) return 1;
    // optimiser step and re-tiling, after every GEMM that read the old weights
    learn_layers(l, net, b, s, pass, grad, scale, st);
    return launch_status(fn);
}
}  // namespace

extern "C" {

int dm_learn_set_weights(dm_learn* l, const dm_learn_net* net, void* stream) {
    return learn<dm_learn_batch>("dm_learn_set_weights", Pass::retile, l, net, nullptr, nullptr, 1.f, stream);
}

int dm_learn_step(dm_learn* l, const dm_learn_net* net, const dm_learn_batch* b, void* stream) {
    return learn("dm_learn_step", Pass::step, l, net, b, nullptr, 1.f, stream);
}

int dm_learn_grad(dm_learn* l, const dm_learn_net* net, const dm_learn_batch* b, float* d_grad, void* stream) {
    return learn("dm_learn_grad", Pass::pack, l, net, b, d_grad, 1.f, stream);
}

int dm_learn_apply(dm_learn* l, const dm_learn_net* net, const dm_learn_batch* b, const float* d_grad, float scale, void* stream) {
    return learn("dm_learn_apply", Pass::apply, l, net, b, const_cast<float*>(d_grad), scale, stream);
}

int dm_learn_disc_step(dm_learn* l, const dm_learn_net* net, const dm_learn_disc_batch* b, void* stream) {
    return learn("dm_learn_disc_step", Pass::step, l, net, b, nullptr, 1.f, stream);
}

int dm_learn_disc_grad(dm_learn* l, const dm_learn_net* net, const dm_learn_disc_batch* b, float* d_grad, void* stream) {
    return learn("dm_learn_disc_grad", Pass::pack, l, net, b, d_grad, 1.f, stream);
}

int dm_learn_disc_apply(dm_learn* l, const dm_learn_net* net, const dm_learn_disc_batch* b, const float* d_grad, float scale, void* stream) {
    return learn("dm_learn_disc_apply", Pass::apply, l, net, b, const_cast<float*>(d_grad), scale, stream);
}

int dm_learn_set_gated_weights(dm_learn* l, const dm_learn_gated_net* net, void* stream) {
    return learn<dm_learn_gated_batch>("dm_learn_set_gated_weights", Pass::retile, l, net, nullptr, nullptr, 1.f, stream);
}

int dm_learn_gated_step(dm_learn* l, const dm_learn_gated_net* net, const dm_learn_gated_batch* gb, void* stream) {
    return learn("dm_learn_gated_step", Pass::step, l, net, gb, nullptr, 1.f, stream);
}

int dm_learn_gated_grad(dm_learn* l, const dm_learn_gated_net* net, const dm_learn_gated_batch* gb, float* d_grad, void* stream) {
    return learn("dm_learn_gated_grad", Pass::pack, l, net, gb, d_grad, 1.f, stream);
}

int dm_learn_gated_apply(dm_learn* l, const dm_learn_gated_net* net, const dm_learn_gated_batch* gb, const float* d_grad, float scale, void* stream) {
    return learn("dm_learn_gated_apply", Pass::apply, l, net, gb, const_cast<float*>(d_grad), scale, stream);
}

int dm_mlp_set_gated_weights_device(dm_mlp* m, const float* const* d_w, const float* const* d_b, void* stream) {
    if (!m) return mlp_fail("dm_mlp_set_gated_weights_device: null handle");
    if (!m->gated) return mlp_fail("dm_mlp_set_gated_weights_device: the handle holds a plain network (dm_mlp_create); use dm_mlp_set_weights_device");
    if (!d_w || !d_b) return mlp_fail("dm_mlp_set_gated_weights_device: null weight pointer");
    for (int i = 0; i < 10; ++i)
        if (!d_w[i] || !d_b[i]) return mlp_fail("dm_mlp_set_gated_weights_device: null weight pointer");
    if (cudaSetDevice(m->device) != cudaSuccess) return mlp_fail("dm_mlp_set_gated_weights_device: cudaSetDevice failed");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    for (int i = 0; i < 10; ++i) launch_layer(gated_layer_params(m, i, d_w[i], d_b[i]), st);
    return launch_status("dm_mlp_set_gated_weights_device");
}

int dm_mlp_set_gated_normalizers_device(dm_mlp* m, const float* d_s_mean, const float* d_s_std, const float* d_g_mean, const float* d_g_std, const float* d_out_mean,
                                        const float* d_out_std, void* stream) {
    if (!m) return mlp_fail("dm_mlp_set_gated_normalizers_device: null handle");
    if (!m->gated) return mlp_fail("dm_mlp_set_gated_normalizers_device: the handle holds a plain network (dm_mlp_create); use dm_mlp_set_normalizers_device");
    if (!d_s_mean || !d_s_std || !d_g_mean || !d_g_std || !d_out_mean || !d_out_std) return mlp_fail("dm_mlp_set_gated_normalizers_device: null normaliser pointer");
    if (cudaSetDevice(m->device) != cudaSuccess) return mlp_fail("dm_mlp_set_gated_normalizers_device: cudaSetDevice failed");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    dmk::dm_learn_norm_kernel<<<(m->in_dim + 255) / 256, 256, 0, st>>>(d_s_mean, d_s_std, m->in_dim, m->in_mean, m->in_istd, 1);
    dmk::dm_learn_norm_kernel<<<(m->goal_dim + 255) / 256, 256, 0, st>>>(d_g_mean, d_g_std, m->goal_dim, m->g_mean, m->g_istd, 1);
    dmk::dm_learn_norm_kernel<<<(m->out_dim + 255) / 256, 256, 0, st>>>(d_out_mean, d_out_std, m->out_dim, m->out_mean, m->out_std, 0);
    return launch_status("dm_mlp_set_gated_normalizers_device");
}

void dm_learn_destroy(dm_learn* l) {
    if (!l) return;
    cudaSetDevice(l->m->device);
    for (void* p : l->bufs) cudaFree(p);
    dm_mlp_destroy(l->m);
    delete l;
}

long long dm_mlp_launches(dm_mlp* m) { return m ? m->launches : 0; }

void dm_mlp_destroy(dm_mlp* m) {
    if (!m) return;
    cudaSetDevice(m->device);
    for (void* p : m->bufs) cudaFree(p);
    delete m;
}

}  // extern "C"
