// Ray-cast rendering of pose rows (dm_render.cu, C ABI dm_render_poses and dm_render_poses_marked): the character's collision shapes on a checkered ground plane, seen
// from a camera that tracks each row's root.
#pragma once
#include <cstdint>

#include "dm_model.cuh"

namespace dmk {

constexpr int kRenderTile = 16;   // dm_render_kernel: one block of 16 x 16 threads per 16 x 16 pixel tile of one view

// the camera of all views, unscaled metres: eye = (root x, target_height, root z) + back; a pixel's ray is fwd + sx right + sy up with
// sx, sy in [-tan_x, tan_x] x [-tan_y, tan_y] at the pixel centre (dm_render_poses derives it from dm_camera in double)
struct RenderCam {
    float back[3], fwd[3], right[3], up[3];
    float tan_x, tan_y, target_height;
};

__global__ void dm_render_kernel(const DevModel* gm, const float* pose, int width, int height, RenderCam cam, uint8_t* rgb, int16_t* ids);
// one marker sphere per view (dm_render_poses_marked), an overlay launched after dm_render_kernel on the same outputs that writes only the
// pixels the marker changes: marker [views x 4] = x, y, z, radius (unscaled metres; radius <= 0: none)
constexpr int kRenderMarkerId = -3;   // the ids value of the marker's pixels
__global__ void dm_render_marked_kernel(const DevModel* gm, const float* pose, const float* marker, int width, int height, RenderCam cam, uint8_t* rgb,
                                        int16_t* ids);

}  // namespace dmk
