// Common definitions for the fiducials_b200 device code.
//
// All per-element logic of the pipeline lives in FID_HD functions so that the *same source* is
// compiled (a) by nvcc into the sm_90a kernels of libfiducials_b200.so (the product) and (b) by
// g++ into tests/hostsim (a CPU unit-test harness for the device functions; never linked into the
// product library, never reachable from the C-ABI).
#pragma once
#include <stdint.h>
#include <math.h>

#if defined(__CUDACC__)
#define FID_HD __host__ __device__ __forceinline__
#define FID_D __device__ __forceinline__
#else
#define FID_HD inline
#define FID_D inline
#endif

namespace fid {

#define FID_MAX_SCALES 16
#define FID_MAX_WIN_RADIUS 31   // adaptive-threshold window <= 63
#define FID_MAX_WARP_SIDE 72    // (markerSize + 2*border) * pixelPerCell: 7x7 markers with the reference's 8 pixels per cell
#define FID_MAX_WARP_SIDE_SQ (FID_MAX_WARP_SIDE * FID_MAX_WARP_SIDE)

struct Pt16 {
    int16_t x, y;
};

FID_HD int fid_clz(uint32_t v) {
#if defined(__CUDA_ARCH__)
    return __clz((int)v);
#else
    return v ? __builtin_clz(v) : 32;
#endif
}
FID_HD int fid_ctz(uint32_t v) {
#if defined(__CUDA_ARCH__)
    return __ffs((int)v) - 1;
#else
    return v ? __builtin_ctz(v) : -1;
#endif
}
FID_HD int fid_popc(uint32_t v) {
#if defined(__CUDA_ARCH__)
    return __popc(v);
#else
    return __builtin_popcount(v);
#endif
}

// cv::cvtColor(BGR2GRAY) of one 8-bit pixel: 15-bit fixed point (SURVEY A.1)
FID_HD uint32_t gray_of_bgr(uint32_t b, uint32_t g, uint32_t r) { return (3735u * b + 19235u * g + 9798u * r + 16384u) >> 15; }

// Gray image accessors for the stages that sample a few pixels (identification, cornerSubPix): either
// a gray plane, or the frame itself in the encoding cv_bridge::toCvCopy(msg, BGR8) was given
// (aruco_detect.cpp:348) -- the tensor-core threshold kernel never writes a gray plane to HBM.
struct GrayPlane {
    const uint8_t* p;
    size_t pitch;
    FID_HD int at(int x, int y) const { return p[(size_t)y * pitch + x]; }
};
struct FrameImg {
    const uint8_t* p;
    size_t row_stride;
    int enc;  // 0 bgr8, 1 rgb8, 2 mono8
    FID_HD int at(int x, int y) const {
        const uint8_t* q = p + (size_t)y * row_stride;
        if (enc == 2) return q[x];
        q += 3 * (size_t)x;
        return (int)(enc == 1 ? gray_of_bgr(q[2], q[1], q[0]) : gray_of_bgr(q[0], q[1], q[2]));
    }
};

// Detector parameters as consumed by the device code.  Mirrors the 21 fields of
// aruco_detect/cfg/DetectorParams.cfg that aruco_detect.cpp:690-727 sets, plus the two OpenCV-4.13
// fields the oracle fixes (SURVEY A.0).
struct DevParams {
    int n_scales;                   // (max-min)/step+1                         (aruco_detect.cpp:691-693)
    int win[FID_MAX_SCALES];        // odd window sizes
    int thresh_c;                   // floor(adaptiveThreshConstant)            (:690)
    double min_perimeter_rate;      // :722
    double max_perimeter_rate;      // :723
    double poly_accuracy_rate;      // :727
    double min_corner_dist_rate;    // :717
    int min_dist_to_border;         // :720
    double min_marker_dist_rate;    // :721
    int marker_border_bits;         // :718
    int px_per_cell;                // :726
    double ignored_margin_per_cell; // :725
    double max_err_border_rate;     // :719
    double min_otsu_stddev;         // :724
    double error_correction_rate;   // :716
    int corner_refine;              // 0 none, 1 subpix                         (:700-711)
    int refine_win;                 // :696
    int refine_max_iter;            // :694
    double refine_min_acc;          // :695
    double rel_refine_win;          // 4.13-only; oracle = 100
    double min_group_dist;          // 4.13-only; 0.21
    // dictionary
    int marker_size;                // 5 or 6
    int n_markers;
    int max_correction_bits;
    int dict_nbytes;                // (ms*ms+7)/8
    int dict_table;                 // index into kDictTables (host side)
};

}  // namespace fid
