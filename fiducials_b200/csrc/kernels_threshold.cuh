// CUDA kernels, threshold stage (sm_90a):
//   k_gray       BGR8 -> gray (cv::cvtColor BGR2GRAY, 15-bit fixed point, SURVEY A.1); 4 pixels per
//                thread, 12-byte vector loads / 4-byte store
//   k_threshold  frame (BGR8/RGB8/MONO8; cvtColor fused into the load) -> n_scales adaptive-threshold planes (SURVEY A.2), written directly as the
//                bit-packed halo tiles the border walk reads (contour_walk.cuh, HaloView), plus the
//                start-crack queues of the border walk (exact local prune) while the tiles are in registers
//
// k_threshold: one CTA per 120x60 output pixels = 4x2 halo tiles.  The CTA loads the gray region it
// needs (output + 1 halo pixel + r_max on every side, replicate border) into shared memory, turns
// it into a summed-area table, and every scale's box sum is 4 look-ups.  BINARY_INV with the mean
// rounded half-to-even (no ties for odd windows) reduces to the integer test
//     2*S >= (2*g + 2*C - 1) * k^2
// A warp covers the 32 bit positions of one tile word, so __ballot_sync IS the word.  With the
// reference's windows 3,7,...,51 the scale loop is unrolled at compile time and every table offset
// is an immediate.
// Algorithmic HBM bytes per frame (SURVEY 8d): 3*W*H in + n_scales*W*H/8 out (+ W*H gray out/in).
#pragma once
#include <cuda_runtime.h>

#include "common.cuh"
#include "contour_walk.cuh"
#include "kernels_threshold_tail.cuh"  // tail shared by both threshold kernels

namespace fid {

struct GrayArgs {
    const uint8_t* bgr;
    uint8_t* gray;
    int W, H, n_frames;
    size_t bgr_row_stride, bgr_frame_stride;
    int gray_pitch;
    size_t gray_frame_stride;
    int enc;  // FID_ENC_*: what cv_bridge::toCvCopy(msg, BGR8) would have been given (aruco_detect.cpp:348)
};

__device__ __forceinline__ uint32_t gray_of(uint32_t b, uint32_t g, uint32_t r) { return gray_of_bgr(b, g, r); }

__global__ void __launch_bounds__(256) k_gray(const GrayArgs a) {
    const int quads = (a.W + 3) >> 2;
    const long long total = (long long)a.n_frames * a.H * quads;
    const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const int q = (int)(gid % quads);
    const long long t = gid / quads;
    const int y = (int)(t % a.H), f = (int)(t / a.H);
    const int x = q * 4;
    uint8_t* dst = a.gray + (size_t)f * a.gray_frame_stride + (size_t)y * a.gray_pitch + x;
    if (a.enc == 2) {  // MONO8: toCvCopy replicates the channel and BGR2GRAY of (g,g,g) is g exactly ((32768 g + 16384) >> 15)
        const uint8_t* src = a.bgr + (size_t)f * a.bgr_frame_stride + (size_t)y * a.bgr_row_stride + (size_t)x;
        if (x + 3 < a.W && ((reinterpret_cast<uintptr_t>(src) & 3) == 0)) {
            *reinterpret_cast<uint32_t*>(dst) = __ldg(reinterpret_cast<const uint32_t*>(src));
        } else {
            for (int k = 0; k < 4 && x + k < a.W; k++) dst[k] = src[k];
        }
        return;
    }
    const uint8_t* src = a.bgr + (size_t)f * a.bgr_frame_stride + (size_t)y * a.bgr_row_stride + 3 * (size_t)x;
    const bool rgb = a.enc == 1;  // RGB8: toCvCopy swaps the channels first, i.e. the first byte is R
    if (x + 3 < a.W && ((reinterpret_cast<uintptr_t>(src) & 3) == 0)) {
        const uint32_t w0 = __ldg(reinterpret_cast<const uint32_t*>(src));      // B0 G0 R0 B1
        const uint32_t w1 = __ldg(reinterpret_cast<const uint32_t*>(src) + 1);  // G1 R1 B2 G2
        const uint32_t w2 = __ldg(reinterpret_cast<const uint32_t*>(src) + 2);  // R2 B3 G3 R3
        uint32_t c0[4] = {w0 & 255u, w0 >> 24, (w1 >> 16) & 255u, (w2 >> 8) & 255u};
        const uint32_t c1[4] = {(w0 >> 8) & 255u, w1 & 255u, w1 >> 24, (w2 >> 16) & 255u};
        uint32_t c2[4] = {(w0 >> 16) & 255u, (w1 >> 8) & 255u, w2 & 255u, w2 >> 24};
        uint32_t out = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) out |= (rgb ? gray_of(c2[k], c1[k], c0[k]) : gray_of(c0[k], c1[k], c2[k])) << (8 * k);
        *reinterpret_cast<uint32_t*>(dst) = out;  // gray_pitch and x are multiples of 4
    } else {
        for (int k = 0; k < 4 && x + k < a.W; k++) {
            const uint32_t p0 = src[3 * k], p1 = src[3 * k + 1], p2 = src[3 * k + 2];
            dst[k] = (uint8_t)(rgb ? gray_of(p2, p1, p0) : gray_of(p0, p1, p2));
        }
    }
}

// ---------------------------------------------------------------------------------------------------
#define THR_TILES_X 4
#define THR_TILES_Y 2
#define THR_OW (THR_TILES_X * FID_HALO_T)  // 120 output columns per CTA
#define THR_OH (THR_TILES_Y * FID_HALO_T)  // 60 output rows per CTA
#define THR_THREADS 256
#define THR_FAST_R 25                      // r_max of the reference's window set

struct ThreshArgs {
    const uint8_t* src;  // the frames as delivered (BGR8 / RGB8 / MONO8): cvtColor is fused into the region load
    size_t src_row_stride, src_frame_stride;
    int enc;
    int aligned4;        // W, the base pointer and both strides are multiples of 4 -> 4-pixel groups with 32-bit loads
    uint32_t* halo;
    int W, H, n_frames;
    int halo_tpr, halo_tiles_y;
    size_t halo_scale_stride, halo_frame_stride;
    int n_scales;
    int r_max;
    int thresh_c;
    int win[FID_MAX_SCALES];
    StartRec* starts;      // start-crack queue: left cracks at [0, nL), right cracks at [max_starts-1 ...]
    Counters* counters;
    unsigned int max_starts;
    const uint32_t* prune;  // kStartPruneTable on the device (FID_START_PRUNE=1) or NULL
};

// gray byte tile: region column rx lives at byte rx + 2 of its row (the 4-pixel groups of the fast load start 2 columns left of the
// region); the pitch is an ODD number of words so that 32 consecutive rows fall into 32 different banks
__host__ __device__ inline int thresh_gray_pitch_words(int r_max) { return ((THR_OW + 2 + 2 * r_max + 2 + 3 + 3) / 4) | 1; }
__host__ __device__ inline size_t thresh_smem_bytes(int r_max) {
    const int RW = THR_OW + 2 + 2 * r_max, RH = THR_OH + 2 + 2 * r_max;
    return (size_t)(RH + 1) * (RW + 1) * 4 + (size_t)RH * thresh_gray_pitch_words(r_max) * 4;
}

// FAST: windows 3 + 4*s (s = 0..12), r_max = 25 -> everything below is compile-time.
#ifndef THR_MAXNREG
#define THR_MAXNREG 96  // 2 CTAs per SM leave a quarter of the register file to the kernels of other chunks (+1 % pipelined, no spills)
#endif
// PRUNE: the opt-in table stage of the start pruning (FID_START_PRUNE=1) is its own instantiation, so that the default kernel is
// instruction for instruction the one that was measured.
template <bool FAST, bool PRUNE = false>
__global__ void __maxnreg__(THR_MAXNREG) k_threshold(const ThreshArgs a) {
    extern __shared__ uint32_t sat[];
    const int R = FAST ? THR_FAST_R : a.r_max;
    const int RW = THR_OW + 2 + 2 * R, RH = THR_OH + 2 + 2 * R;
    const int SP = RW + 1;  // table pitch; row 0 / column 0 are zero
    const int GPW = FAST ? thresh_gray_pitch_words(THR_FAST_R) : thresh_gray_pitch_words(a.r_max);
    uint32_t* gbw = sat + (RH + 1) * SP;                      // gray byte tile, RH rows of GPW words
    uint8_t* gb = reinterpret_cast<uint8_t*>(gbw);
    const int f = blockIdx.z;
    const int X0 = blockIdx.x * THR_OW, Y0 = blockIdx.y * THR_OH;  // first output pixel of the CTA
    const int W = a.W, H = a.H;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint8_t* src = a.src + (size_t)f * a.src_frame_stride;

    for (int i = tid; i < SP; i += THR_THREADS) sat[i] = 0;
    for (int i = tid; i <= RH; i += THR_THREADS) sat[i * SP] = 0;
    // A. gray region (replicate border): region (0,0) = image (X0-1-R, Y0-1-R).  cv::cvtColor BGR2GRAY happens here, on the
    //    way from global to shared memory: the gray plane is never written to or read back from HBM.
    const int XA = X0 - 1 - R - 2;  // multiple of 4 when R = 25 (X0 is a multiple of 120): region column c = group column 4w - 2 + b
    if (FAST && a.aligned4) {
        // 4-pixel groups, 32-bit loads (3 words of BGR, or 1 word of MONO8).  XA and W are multiples of 4, so a group lies either
        // inside the image or entirely left / right of it: outside groups replicate the first / last pixel of the clamped group.
        // Thread (w, r0) of the first 5 x 44 threads owns group column w and the rows r0, r0 + 5, ...: no divisions, a pointer
        // step per row, store predicates that depend on w only.  Gray = two byte dot products per pixel (IDP4A) with the 15-bit
        // cvtColor coefficients split into high and low bytes: sum p*c = 256 * sum p*c_hi + sum p*c_lo, exactly.
        constexpr int GPR = (THR_OW + 2 + 2 * THR_FAST_R + 2 + 3) / 4;  // 44 groups per row
        constexpr int RHc = THR_OH + 2 + 2 * THR_FAST_R;                  // 112 rows
        constexpr int RPP = THR_THREADS / GPR;                            // 5 rows per pass
        constexpr int CH = 6;                                             // passes in flight per thread (18 words)
        if (tid < RPP * GPR) {
            const int r0 = tid / GPR, w = tid - r0 * GPR;
            const int gmax = (W >> 2) - 1;
            const int gx = (XA >> 2) + w;
            const int gxc = gx < 0 ? 0 : (gx > gmax ? gmax : gx);
            const bool left = gx < 0, right = gx > gmax;
            const bool mono = a.enc == 2;
            // coefficient words for the pixels at byte offsets 0 (and the two re-assembled pixels) and 1 of a word
            const uint32_t cb = 3735u, cg = 19235u, cr = 9798u;
            const uint32_t c0 = a.enc == 1 ? cr : cb, c2 = a.enc == 1 ? cb : cr;  // RGB8: the first byte is R
            const uint32_t lo0 = (c0 & 255u) | ((cg & 255u) << 8) | ((c2 & 255u) << 16), hi0 = (c0 >> 8) | ((cg >> 8) << 8) | ((c2 >> 8) << 16);
            const uint32_t lo1 = lo0 << 8, hi1 = hi0 << 8;
            const uint8_t* colp = src + (mono ? 4 : 12) * (size_t)gxc;
            uint32_t* gcol = gbw + w;  // the group's four gray bytes are ONE word of the byte tile: conflict-free 32-bit stores
#pragma unroll 1
            for (int rb = r0; rb < RHc; rb += CH * RPP) {
                uint32_t v[CH][3];
#pragma unroll
                for (int k = 0; k < CH; k++) {
                    const int ry = rb + k * RPP;
                    int y = Y0 - 1 - R + ry;
                    y = y < 0 ? 0 : (y > H - 1 ? H - 1 : y);
                    const uint32_t* q = reinterpret_cast<const uint32_t*>(colp + (size_t)y * a.src_row_stride);
                    if (ry < RHc) {
                        v[k][0] = __ldg(q);
                        if (!mono) {
                            v[k][1] = __ldg(q + 1);
                            v[k][2] = __ldg(q + 2);
                        }
                    }
                }
#pragma unroll
                for (int k = 0; k < CH; k++) {
                    const int ry = rb + k * RPP;
                    if (ry < RHc) {
                        uint32_t g0, g1, g2, g3;
                        if (mono) {
                            g0 = v[k][0] & 255u;
                            g1 = (v[k][0] >> 8) & 255u;
                            g2 = (v[k][0] >> 16) & 255u;
                            g3 = v[k][0] >> 24;
                        } else {
                            const uint32_t w0 = v[k][0], w1 = v[k][1], w2 = v[k][2];  // B0 G0 R0 B1 | G1 R1 B2 G2 | R2 B3 G3 R3
                            const uint32_t p1 = __byte_perm(w0, w1, 0x5543), p2 = __byte_perm(w1, w2, 0x4432);
                            g0 = (__dp4a(w0, lo0, 16384u) + (__dp4a(w0, hi0, 0u) << 8)) >> 15;
                            g1 = (__dp4a(p1, lo0, 16384u) + (__dp4a(p1, hi0, 0u) << 8)) >> 15;
                            g2 = (__dp4a(p2, lo0, 16384u) + (__dp4a(p2, hi0, 0u) << 8)) >> 15;
                            g3 = (__dp4a(w2, lo1, 16384u) + (__dp4a(w2, hi1, 0u) << 8)) >> 15;
                        }
                        if (left) g1 = g2 = g3 = g0;
                        if (right) g0 = g1 = g2 = g3;
                        gcol[ry * GPW] = g0 | (g1 << 8) | (g2 << 16) | (g3 << 24);
                    }
                }
            }
        }
    } else {
        const FrameImg img{src, a.src_row_stride, a.enc};
        for (int ry = warp; ry < RH; ry += THR_THREADS / 32) {
            int y = Y0 - 1 - R + ry;
            y = y < 0 ? 0 : (y > H - 1 ? H - 1 : y);
            uint8_t* grow = gb + (size_t)ry * GPW * 4 + 2;
            for (int rx = lane; rx < RW; rx += 32) {
                int x = X0 - 1 - R + rx;
                x = x < 0 ? 0 : (x > W - 1 ? W - 1 : x);
                grow[rx] = (uint8_t)img.at(x, y);
            }
        }
    }
    __syncthreads();
    // B. row prefix sums: one thread per row reads the row's gray bytes four at a time and writes the running sums into the table
    //    (both conflict free: rows are an odd number of words apart in either array)
    for (int ry = tid; ry < RH; ry += THR_THREADS) {
        uint32_t* row = sat + (ry + 1) * SP + 1;
        const uint32_t* gw = gbw + ry * GPW;
        uint32_t acc = 0;
        {
            const uint32_t v = gw[0];  // bytes 2, 3 = region columns 0, 1
            acc += (v >> 16) & 255u;
            row[0] = acc;
            acc += v >> 24;
            row[1] = acc;
        }
        int c = 2;
#pragma unroll 4
        for (int j = 1; c + 4 <= RW; j++, c += 4) {
            const uint32_t v = gw[j];
            const uint32_t v0 = v & 255u, v1 = (v >> 8) & 255u, v2 = (v >> 16) & 255u, v3 = v >> 24;
            row[c] = acc + v0;
            row[c + 1] = acc + v0 + v1;
            row[c + 2] = acc + v0 + v1 + v2;
            acc += v0 + v1 + v2 + v3;
            row[c + 3] = acc;
        }
        if (c < RW) {
            const uint32_t v = gw[(c + 2) >> 2];
            for (int b = 0; c < RW; c++, b++) {
                acc += (v >> (8 * b)) & 255u;
                row[c] = acc;
            }
        }
    }
    __syncthreads();
    // C. column prefix sums: one thread per column
    for (int c = tid; c < RW; c += THR_THREADS) {
        uint32_t acc = 0;
        uint32_t* col = sat + SP + 1 + c;
        for (int ry = 0; ry < RH; ry++) {
            acc += col[ry * SP];
            col[ry * SP] = acc;
        }
    }
    __syncthreads();
    // D. one warp per halo tile: lane = bit position (column), loop over the 32 rows of the tile; lane r
    //    keeps the word of row r for every scale, so at the end the warp holds the 13 finished tiles in
    //    registers: one coalesced 128-byte store per scale, and the start cracks of the border walk
    //    (contour_walk.cuh, halo_row_starts) come from two shuffles -- the planes are never read back.
    //    Test: 2S >= (2g + 2C - 1) k^2 with an odd right-hand side  <=>  S >= g k^2 + ((2C-1) k^2 + 1)/2.
    constexpr int NS = FAST ? 13 : FID_MAX_SCALES;
    const int twoC = 2 * a.thresh_c - 1;
    const int txl = warp % THR_TILES_X, tyl = warp / THR_TILES_X;
    const int tx = blockIdx.x * THR_TILES_X + txl, ty = blockIdx.y * THR_TILES_Y + tyl;
    if (tx >= a.halo_tpr || ty >= a.halo_tiles_y) return;  // warp-uniform; no block barrier below
    // Orientation: lane = tile ROW, the loop runs over the 32 columns from the last to the first and shifts the result bit of
    // (row lane, column c) into the lane's word -- no ballot, no select, and lane r ends with the word of row r as the tail
    // expects.  Lanes are SP = 173 words apart: 13 r mod 32 is a bijection, the loads are conflict free.  The test is folded
    // into one sign bit: nd = g k^2 + (ck - 1) - S < 0  <=>  S >= g k^2 + ck; per pixel and scale that is 4 loads, 2 IADD3,
    // 1 IMAD and 1 funnel shift.
    uint32_t acc[NS];
    int kk[NS], ckm1[NS], off_br[NS], off_bl[NS], off_tr[NS], off_tl[NS];
#pragma unroll
    for (int s = 0; s < NS; s++) {
        acc[s] = 0;
        const int k = FAST ? 3 + 4 * s : (s < a.n_scales ? a.win[s] : 1), rr = k >> 1;
        kk[s] = k * k;
        ckm1[s] = (twoC * k * k + 1) / 2 - 1;  // exact: odd * odd + 1 is even
        off_br[s] = (rr + 1) * SP + rr + 1;
        off_bl[s] = (rr + 1) * SP - rr;
        off_tr[s] = -rr * SP + rr + 1;
        off_tl[s] = -rr * SP - rr;
    }
    {
        const uint32_t* prow = sat + (FID_HALO_T * tyl + R + lane) * SP + (FID_HALO_T * txl + R);  // table entry "above-left" of (row lane, column 0)
        const uint8_t* grow = gb + (size_t)(FID_HALO_T * tyl + R + lane) * GPW * 4 + (FID_HALO_T * txl + R) + 2;
#pragma unroll 1
        for (int c = 31; c >= 0; c--) {
            const uint32_t* p = prow + c;
            const int g = grow[c];  // the pixel itself: one byte load instead of four table look-ups
#pragma unroll
            for (int s = 0; s < NS; s++) {
                if (!FAST && s >= a.n_scales) break;
                const int t = g * kk[s] + ckm1[s];
                const int u = t + (int)p[off_bl[s]] + (int)p[off_tr[s]];
                const int nd = u - (int)p[off_br[s]] - (int)p[off_tl[s]];
                acc[s] = __funnelshift_l((uint32_t)nd, acc[s], 1);
            }
        }
        // pixels outside the image are background
        const int Xb = X0 + FID_HALO_T * txl - 1, Y = Y0 + FID_HALO_T * tyl - 1 + lane;
        uint32_t colmask = 0xffffffffu;
        if (Xb < 0) colmask &= 0xffffffffu << (-Xb);
        if (Xb + 32 > W) colmask &= W - Xb > 0 ? 0xffffffffu >> (Xb + 32 - W) : 0u;
        if (Y < 0 || Y >= H) colmask = 0u;
#pragma unroll
        for (int s = 0; s < NS; s++) acc[s] &= colmask;
    }
    thr_store_tile_and_starts<NS, PRUNE>(acc, FAST ? 13 : a.n_scales, f, tx, ty, lane, a.halo, a.halo_frame_stride, a.halo_scale_stride, a.halo_tpr, a.halo_tiles_y, a.starts, a.counters,
                                  a.max_starts, a.prune);
}

}  // namespace fid
