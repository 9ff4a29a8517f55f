// TD(lambda) returns and advantages of a batched rollout window (R/learning/rl_util.py: compute_return; R/learning/ppo_agent.py:
// _compute_batch_vals), on the device.  Inputs are [T x N] row major (step-major, environment-minor, as BatchedRollout.collect records them):
//   rewards r, values v = V(s_k), end_values e = V(s'_k) with s'_k the state after step k before the reset, done, terminate (0 null, 1 fail, 2 succ).
// One thread per environment scans k = T - 1 .. 0:
//   v_next = done[k] ? (fail ? val_fail : succ ? val_succ : e[k]) : e[k]
//   G_next = (done[k] || k == T - 1) ? v_next : ret[k + 1]
//   ret[k] = r[k] + gamma ((1 - lambda) v_next + lambda G_next),   adv[k] = ret[k] - v[k].
// When !done[k], e[k] = V(s_{k+1}), so the scan carries nothing but ret[k + 1].  Consecutive threads read consecutive environments of a step, so
// every access is coalesced.  A window has few environments per SM (4096 threads in all), so the scan is bound by load latency: the loads of
// kSteps steps are issued together, before the arithmetic that carries the return through them.
#include <cuda_runtime.h>

#include <cstdint>

#include "dm_mlp.cuh"

namespace dmk {

constexpr int kReturnSteps = 16;   // steps whose loads are in flight at once per thread

__global__ void __launch_bounds__(64) dm_td_lambda_kernel(const float* __restrict__ rewards, const float* __restrict__ values, const float* __restrict__ end_values,
                                                         const uint8_t* __restrict__ done, const int32_t* __restrict__ terminate, int T, int N, float gamma,
                                                         float lambda, float val_fail, float val_succ, float* __restrict__ returns, float* __restrict__ advantages) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    float ret = 0.f;
    for (int k0 = T - 1; k0 >= 0; k0 -= kReturnSteps) {
        float r[kReturnSteps], v[kReturnSteps], e[kReturnSteps];
        uint8_t d[kReturnSteps];
        int32_t tm[kReturnSteps];
#pragma unroll
        for (int u = 0; u < kReturnSteps; ++u) {
            const int k = k0 - u;
            if (k >= 0) {
                const size_t i = static_cast<size_t>(k) * N + n;
                r[u] = rewards[i]; v[u] = values[i]; e[u] = end_values[i]; d[u] = done[i]; tm[u] = terminate[i];
            }
        }
#pragma unroll
        for (int u = 0; u < kReturnSteps; ++u) {
            const int k = k0 - u;
            if (k >= 0) {
                const bool end = d[u] != 0;
                float v_next = e[u];
                if (end && tm[u] == 1) v_next = val_fail;
                if (end && tm[u] == 2) v_next = val_succ;
                const float g_next = (end || k == T - 1) ? v_next : ret;
                ret = r[u] + gamma * ((1.f - lambda) * v_next + lambda * g_next);
                const size_t i = static_cast<size_t>(k) * N + n;
                returns[i] = ret;
                advantages[i] = ret - v[u];
            }
        }
    }
}

}  // namespace dmk
