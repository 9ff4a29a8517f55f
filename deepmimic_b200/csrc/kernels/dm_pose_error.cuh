// How closely pose rows follow a reference (dm_pose_error.cu, C ABI dm_pose_error): per episode the phase-locked and the dynamic-time-warped
// mean joint-position error, in the character's heading frame.
#pragma once
#include <cstdint>

#include "dm_model.cuh"

namespace dmk {

constexpr int kPoseFeatureThreads = 256;   // dm_pose_feature_kernel: one warp per pose row
constexpr int kPoseDtwThreads = 128;       // dm_pose_dtw_kernel: one block per episode, one thread per row of a strip of the DP grid
static_assert(3 * (kMaxLinks - 1) <= kPoseDtwThreads, "one thread per feature component loads the reference's next frame");

// features [2][n][T][3 (nl - 1)]: of the rows a (blockIdx.y 0) and r (1), [T][n][pose_dim] each
__global__ void dm_pose_feature_kernel(const DevModel* gm, const float* a, const float* r, int T, int n, float* feat);
// dm_pose_dtw_kernel<NJ>: lock / dtw [n] (either may be null), bnd [n][T] scratch; [0]: NJ = 15 joints besides the root at most, [1]: 31
using PoseDtwKernel = void (*)(const float* feat, int T, int n, int nj, const int32_t* len, float* bnd, float* lock, float* dtw);
extern const PoseDtwKernel kPoseDtwKernels[2];
// bytes of dynamic shared memory of dm_pose_dtw_kernel: the reference frames' ring
inline size_t dm_pose_dtw_smem(int nj) { return sizeof(float) * 3 * nj * 2 * kPoseDtwThreads; }

}  // namespace dmk
