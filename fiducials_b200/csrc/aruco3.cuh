// useAruco3Detection of cv::aruco::ArucoDetector (OpenCV 4.13; Romero-Ramirez et al. 2018, "Speeded up detection of squared
// fiducial markers"), DESIGN.md finding 16.  Segmentation runs on the gray frame scaled by
//     fxfy = minSide / (minSide + max(W, H) * ratio)                                  (float32)
// with cv::resize(INTER_LINEAR); the bits of each candidate are read from the pyramid level (buildPyramid, pyrDown) whose scaled
// contour length is closest above 4 * minSide; the corners are scaled to level `closest` and refined by cornerSubPix on every
// finer level.  The per-pixel functions below are bit-exact with cv2.resize / cv2.pyrDown and are compiled both into the
// kernels (kernels_aruco3.cuh) and into the CPU harness (tests/hostsim/aruco3_hostsim.cpp).
#pragma once
#include <float.h>

#include "common.cuh"
#include "quad_group.cuh"
#include "subpix.cuh"

namespace fid {

#define FID_ARUCO3_MAX_LEVELS 16  // a 16384 x 16384 frame with minSide 1 has 15 pyramid images

struct A3Level {
    size_t off;  // byte offset of the level in a frame's pyramid block (levels >= 1; level 0 is the gray plane)
    int W, H, pitch;
};

// The per-frame-size geometry of the mode (host computed, passed to the kernels by value).
struct A3Geom {
    int W, H;          // full resolution
    int seg_w, seg_h;  // segmentation plane
    int n_levels;      // pyramid images, level 0 included (buildPyramid's maxlevel + 1)
    int closest;       // level the corners are scaled to before the cornerSubPix passes
    int min_side;      // minSideLengthCanonicalImg
    int resized;       // fxfy != 1: the segmentation plane is a resized copy, else the gray plane itself
    float fxfy;
    A3Level lv[FID_ARUCO3_MAX_LEVELS];
    size_t pyr_frame_bytes;  // levels 1 .. n_levels - 1 of one frame
};

// The pyramid of a batch on the device: level 0 is the gray plane (pitch lv[0].pitch), levels >= 1 lie in one block per frame.
struct A3Pyramid {
    const uint8_t* gray;
    size_t gray_frame_stride;
    const uint8_t* pyr;
    const RawQuad* raw;  // [F][max_raw]: the contour lengths that pick a candidate's level
    A3Geom g;
    FID_HD GrayPlane plane(int f, int l) const {
        return l == 0 ? GrayPlane{gray + (size_t)f * gray_frame_stride, (size_t)g.lv[0].pitch} : GrayPlane{pyr + (size_t)f * g.pyr_frame_bytes + g.lv[l].off, (size_t)g.lv[l].pitch};
    }
};

// ArucoDetector::detectMarkers, steps 0 and 1.1: the scale factor, the pyramid depth and the level closest to the segmentation
// plane.  All in float32 as cv2 computes them.  Returns false when the pyramid would be deeper than FID_ARUCO3_MAX_LEVELS.
inline bool a3_geometry(int W, int H, int min_side, double ratio, A3Geom* g) {
    const float fr = (float)ratio;
    const float fxfy = (float)min_side / ((float)min_side + (float)(W > H ? W : H) * fr);
    const float img_area = (float)(W * H);
    const float min_area = (float)(min_side * min_side);
    const int num_levels = (int)(log2(img_area / min_area) / 2.f);
    const float scale_area = img_area * fxfy * fxfy;
    const int closest = (int)nearbyint(log2(img_area / scale_area) / 2.f);
    if (num_levels + 1 > FID_ARUCO3_MAX_LEVELS || num_levels < 0) return false;
    g->W = W;
    g->H = H;
    g->fxfy = fxfy;
    g->resized = fxfy != 1.f;
    g->seg_w = g->resized ? (int)nearbyintf(fxfy * (float)W) : W;
    g->seg_h = g->resized ? (int)nearbyintf(fxfy * (float)H) : H;
    g->n_levels = num_levels + 1;
    g->closest = closest < num_levels ? closest : num_levels;  // cv2 indexes past the pyramid otherwise; never seen with ratio <= 1
    g->min_side = min_side;
    size_t off = 0;
    int w = W, h = H;
    for (int l = 0; l < g->n_levels; l++) {
        g->lv[l].W = w;
        g->lv[l].H = h;
        g->lv[l].pitch = l == 0 ? (w + 31) / 32 * 32 : w;
        g->lv[l].off = l == 0 ? 0 : off;
        if (l > 0) off += (size_t)w * h;
        w = (w + 1) / 2;
        h = (h + 1) / 2;
    }
    g->pyr_frame_bytes = off;
    return true;
}

FID_HD int a3_reflect101(int i, int n) {
    if (n == 1) return 0;
    while (i < 0 || i >= n) i = i < 0 ? -i : 2 * n - 2 - i;
    return i;
}

// cv::pyrDown (5x5 binomial, BORDER_REFLECT_101, (sum + 128) >> 8) at destination pixel (x, y) of a W x H source.
template <class Img>
FID_HD int a3_pyr_down_at(const Img& src, int W, int H, int x, int y) {
    const int k[5] = {1, 4, 6, 4, 1};
    int xs[5];
    for (int d = 0; d < 5; d++) xs[d] = a3_reflect101(2 * x + d - 2, W);
    int sum = 0;
    for (int dy = 0; dy < 5; dy++) {
        const int sy = a3_reflect101(2 * y + dy - 2, H);
        int row = 0;
        for (int d = 0; d < 5; d++) row += k[d] * src.at(xs[d], sy);
        sum += k[dy] * row;
    }
    return (sum + 128) >> 8;
}

// cv::resize(INTER_LINEAR) coefficients of destination index d (source size sn, scale = 1 / (dn / sn) in double): source index and
// the two 11-bit weights, as resizeGeneric_ computes them.
FID_HD void a3_linear_coef(int d, double scale, int sn, int* s, int* a0, int* a1) {
    float f = (float)((d + 0.5) * scale - 0.5);
    int si = (int)floorf(f);
    f -= (float)si;
    if (si < 0) {
        f = 0.f;
        si = 0;
    }
    if (si >= sn - 1) {
        f = 0.f;
        si = sn - 1;
    }
    *s = si;
    *a0 = (int)nearbyintf((1.f - f) * 2048.f);
    *a1 = (int)nearbyintf(f * 2048.f);
}

// cv::resize(INTER_LINEAR) of an 8-bit plane at destination pixel (x, y).  The horizontal pass is exact in int; the vertical pass is
// the one of OpenCV's vector kernel (VResizeLinearVec_32s8u: both rows >> 4, multiplied high by the 11-bit weights, + 2 >> 2), which
// cv2 runs over whole rows, its scalar formula ((S0 b0 + S1 b1 + 2^21) >> 22) differs in the last bit.
template <class Img>
FID_HD int a3_resize_at(const Img& src, int sw, int sh, double scale_x, double scale_y, int x, int y) {
    int sx, ax0, ax1, sy, ay0, ay1;
    a3_linear_coef(x, scale_x, sw, &sx, &ax0, &ax1);
    a3_linear_coef(y, scale_y, sh, &sy, &ay0, &ay1);
    const int sx1 = sx + 1 < sw ? sx + 1 : sw - 1, sy1 = sy + 1 < sh ? sy + 1 : sh - 1;
    const int s0 = src.at(sx, sy) * ax0 + src.at(sx1, sy) * ax1;
    const int s1 = src.at(sx, sy1) * ax0 + src.at(sx1, sy1) * ax1;
    const int v = ((((s0 >> 4) * ay0) >> 16) + (((s1 >> 4) * ay1) >> 16) + 2) >> 2;
    return v < 0 ? 0 : (v > 255 ? 255 : v);
}

// _findOptPyrImageForCanonicalImg: the level whose scaled contour length exceeds 4 * minSide by the least; level 0 if none does.
FID_HD int a3_level_for(const A3Geom& g, int contour_len) {
    const int min_perimeter = 4 * g.min_side;
    int opt = 0;
    float dist = FLT_MAX;
    for (int i = 0; i < g.n_levels; i++) {
        const float scale = (float)g.lv[i].W / (float)g.seg_w;
        const float nd = (float)contour_len * scale - (float)min_perimeter;
        if (nd < dist && nd > 0.f) {
            dist = nd;
            opt = i;
        }
    }
    return opt;
}

FID_HD float a3_level_scale(const A3Geom& g, int level) { return (float)g.lv[level].W / (float)g.seg_w; }

// findCornerInPyrImage for one corner in segmentation-plane coordinates: scaled to level `closest`, then doubled and refined by
// cornerSubPix (window 5 above 1080 px on the larger side, else 3; zeroZone (-1, -1)) on every finer level.  plane(l) returns the
// level's image; mask(win) the (2 win + 1)^2 weights.
template <class PlaneOf, class MaskOf>
FID_HD void a3_upsample_corner(const A3Geom& g, const PlaneOf& plane, const MaskOf& mask, int max_iters, double eps_sq, float* x, float* y, float* patch) {
    const float s = a3_level_scale(g, g.closest);
    float cx = *x, cy = *y;
    if (s != 1.f) {
        cx *= s;
        cy *= s;
    }
    for (int l = g.closest - 1; l >= 0; l--) {
        cx *= 2.f;
        cy *= 2.f;
        const int win = (g.lv[l].W > g.lv[l].H ? g.lv[l].W : g.lv[l].H) > 1080 ? 5 : 3;
        corner_subpix(plane(l), g.lv[l].W, g.lv[l].H, &cx, &cy, win, mask(win), max_iters, eps_sq, patch);
    }
    *x = cx;
    *y = cy;
}

}  // namespace fid
