// CUDA kernels of useAruco3Detection (aruco3.cuh, DESIGN.md finding 16), sm_90a:
//   k_a3_pyr_down  one pyramid level from the one above it (cv::pyrDown), every frame of a chunk, one thread per output pixel
//   k_a3_resize    the segmentation plane from the gray plane (cv::resize INTER_LINEAR), one thread per output pixel
//   k_a3_corners   findCornerInPyrImage for every corner k_finish wrote (segmentation-plane coordinates -> full resolution)
// The gray plane itself is k_gray's; the stages from the threshold kernel to k_finish run unchanged on the segmentation plane.
#pragma once
#include <cuda_runtime.h>

#include "aruco3.cuh"
#include "kernels_marker.cuh"

namespace fid {

struct A3PlaneArgs {
    const uint8_t* src;
    size_t src_pitch, src_frame_stride;
    int sw, sh;
    uint8_t* dst;
    size_t dst_pitch, dst_frame_stride;
    int dw, dh;
    int n_frames;
    double scale_x, scale_y;  // k_a3_resize: 1 / (dw / sw), 1 / (dh / sh)
};

__global__ void __launch_bounds__(256) k_a3_pyr_down(const A3PlaneArgs a) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, f = blockIdx.z;
    if (x >= a.dw) return;
    const GrayPlane src{a.src + (size_t)f * a.src_frame_stride, a.src_pitch};
    a.dst[(size_t)f * a.dst_frame_stride + (size_t)y * a.dst_pitch + x] = (uint8_t)a3_pyr_down_at(src, a.sw, a.sh, x, y);
}

__global__ void __launch_bounds__(256) k_a3_resize(const A3PlaneArgs a) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, f = blockIdx.z;
    if (x >= a.dw) return;
    const GrayPlane src{a.src + (size_t)f * a.src_frame_stride, a.src_pitch};
    a.dst[(size_t)f * a.dst_frame_stride + (size_t)y * a.dst_pitch + x] = (uint8_t)a3_resize_at(src, a.sw, a.sh, a.scale_x, a.scale_y, x, y);
}

struct A3CornerArgs {
    A3Pyramid pyr;
    const int32_t* count;  // [F]
    float* corners;        // [F][max_markers][8], rewritten in place
    int max_markers;
    const float* subpix_masks;  // k_finish's table: windows 1..5
    int max_iters;
    double eps_sq;
};

// One block per frame, one thread per corner.  The poses follow in k_recovered_pose, over all of the frame's markers.
__global__ void __launch_bounds__(FINISH_THREADS) k_a3_corners(const A3CornerArgs a) {
    const int f = blockIdx.x;
    const int n = a.count[f];
    float* oc = a.corners + (size_t)f * a.max_markers * 8;
    auto plane = [&](int l) { return a.pyr.plane(f, l); };
    auto mask = [&](int win) { return a.subpix_masks + subpix_mask_offset(win); };
    for (int c = threadIdx.x; c < 4 * n; c += FINISH_THREADS) {
        float patch[(2 * FID_SUBPIX_MAX_WIN + 3) * (2 * FID_SUBPIX_MAX_WIN + 3)];
        float x = oc[2 * c], y = oc[2 * c + 1];
        a3_upsample_corner(a.pyr.g, plane, mask, a.max_iters, a.eps_sq, &x, &y, patch);
        oc[2 * c] = x;
        oc[2 * c + 1] = y;
    }
}

}  // namespace fid
