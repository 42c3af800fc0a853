// Threshold stage on the Hopper tensor cores (sm_90a): wgmma u8 x u8 -> s32 + TMA + mbarrier.
//
// Replaces the 13 cv::adaptiveThreshold passes inside cv::aruco::detectMarkers
// (aruco_detect/src/aruco_detect.cpp:350, windows :691-693) and the cvtColor before them, for the
// reference's window set 3,7,...,51.  Same results as kernels_threshold.cuh (bit-exact planes, same
// start cracks); the arithmetic is reorganised so that the adds run on the tensor cores:
//
//   box sum S_r(x,y) = sum_{dy=-r..r} H_r(x, y+dy),   H_r(x,y') = sum_{dx=-r..r} g(x+dx, y')
//
// * H_r for a whole tile is ONE banded matrix product  D[x][y'] = sum_i A_r[x][i] * G[y'][i]
//   (A_r = 0/1 band, u8; G = gray region, u8; exact s32 accumulators in registers):
//   wgmma.mma_async m64n112k32 .s32.u8.u8, two warpgroups of M = 64 output columns each, N = 112
//   region rows, K = 192 region columns (the 4 k-steps that cover the band of the warpgroup's columns).
//   With the rows in REVERSED column order the band matrix is a Hankel matrix (entry depends on
//   row + i only), so its 8x16-byte core matrices are shared along the anti-diagonals: a whole
//   128 x 192 operand is a 38-core-matrix (4.9 KB) table addressed with SBO = 128 B, LBO = 256 B;
//   the second warpgroup starts 8 core matrices (1 KB) into it.
// * The vertical part is a running sum in registers.  Each warpgroup parks its accumulators in shared
//   memory as u16 (H_r <= 51 * 255), one column per 114-entry row; an epilogue thread then owns one
//   column and one 32-row band, streams H_r(x, .) back (leading and trailing edge of the window)
//   and spends three integer operations per pixel and scale:  D = g*(-k^2) + V,  the sign of D into
//   the column word,  V += lead - trail.  The wgmma chain of the next scale is issued before this loop but
//   completes before it starts: it is issued on a conditional path, and ptxas waits for it where the paths
//   join.  Keeping it in flight across the loop (last scale peeled off, issue unconditional) measured 2.5 %
//   slower on H100, the larger code costing more than the overlap gains.  Two parking buffers per
//   warpgroup let a scale be parked while slower threads still read the previous one.  The centre pixels g
//   come straight from the gray tile.
// * BGR tiles are staged by TMA (cp.async.bulk.tensor.3d over a u32 view of the BGR rows, 16-row
//   bands, 4-deep mbarrier ring) and converted to gray in shared memory -- no gray plane in HBM.
//   Tiles whose region leaves the image take a clamping global-load path (replicate border, which
//   TMA's zero fill cannot express): 22 % of the tiles at 1080p.
// * One persistent CTA per SM, warp specialised: warp 0 TMA producer, warps 4-7 BGR->gray converters
//   (they write the MMA's B operand), warps 8-15 the two MMA + epilogue warpgroups, which leave column
//   words in shared memory; the converter warps take them from there while the next tile runs, one
//   warp per two 30x30 halo tiles: 32x32 bit transposes (column words -> row words), the 128-byte tile
//   stores and the start cracks of the border walk, exactly as in kernels_threshold.cuh.
// Algorithmic HBM bytes per frame (SURVEY 8d): 3*W*H in + 13*W*H/8 out.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include "common.cuh"
#include "contour_walk.cuh"
#include "kernels_threshold.cuh"

namespace fid {

#define TM_THREADS 512       // 4 warpgroups: {TMA, 3 idle}, 4 converters, 2 x 4 MMA + epilogue
#define TM_WARP_TMA 0
#define TM_WARP_CONV0 4
#define TM_NCONV 4
#define TM_WARP_EPI0 8
#define TM_NEPI 8
#define TM_START_BLOCK 2048  // start-queue records a warp reserves per global atomic
// registers per thread after setmaxnreg.  The pool is what the CTA was launched with (512 threads -> 128 each), NOT the SM's
// free registers: the four warpgroup values must sum to <= 512 or setmaxnreg.inc spins forever.
#define TM_REGS_CTRL 40
#define TM_REGS_CONV 104
#define TM_REGS_EPI 184
static_assert(TM_REGS_CTRL + TM_REGS_CONV + 2 * TM_REGS_EPI <= 4 * 128, "setmaxnreg budget");
#define TM_N 112      // region rows (MMA N)
#define TM_K 192      // region columns in bytes (6 k-steps of 32)
#define TM_B_LBO (TM_N * 16)          // row-contiguous B tile: (n, i) at (i/16)*TM_B_LBO + n*16 + i%16
#define TM_B_BYTES (12 * TM_B_LBO)    // 21504
#define TM_A_BYTES (38 * 128)         // one Hankel table
#define TM_NTAB 13                    // the 13 window radii
#define TM_C0 154                     // band: A[m][i] = |i + m - 154| <= r   (m = 127 - (x - (X0-1)), i = x - (X0-28))
#define TM_BOXW 148                   // u32 per staged BGR row: 592 B >= 3*(180 + 12); 148 mod 32 = 20 keeps the converters' loads conflict-free
#define TM_BOXH 16
#define TM_NBANDS 7
#define TM_STAGE_BYTES (TM_BOXW * TM_BOXH * 4)
#define TM_STAGE_STRIDE (TM_STAGE_BYTES + 128)  // the converters read up to 5 words past the last row of a box (columns nobody uses): keep them inside the stage
#define TM_NSTAGES 4
#define TM_COLW_WORDS (13 * 2 * 128)
#define TM_OFF_A 0
#define TM_OFF_B (TM_OFF_A + TM_NTAB * TM_A_BYTES)
#define TM_OFF_STAGE (TM_OFF_B + 2 * TM_B_BYTES)
#define TM_OFF_COLW (TM_OFF_STAGE + TM_NSTAGES * TM_STAGE_STRIDE)
// parked accumulators: per warpgroup two buffers of 64 columns x TM_DSTRIDE u16 (region rows 0..111).  57 words per
// column (odd): the 32 columns a warp reads at one row fall in 32 different banks
#define TM_DSTRIDE 114
#define TM_D_BYTES (64 * TM_DSTRIDE * 2)
#define TM_OFF_D (TM_OFF_COLW + 2 * TM_COLW_WORDS * 4)
#define TM_OFF_BAR (TM_OFF_D + 4 * TM_D_BYTES)
#define TM_SMEM_BYTES (TM_OFF_BAR + 256)
static_assert(TM_SMEM_BYTES <= 227 * 1024, "H100: at most 227 KB of shared memory per block");

// barrier indices (uint64 each)
enum { TMB_STAGE_FULL = 0, TMB_STAGE_EMPTY = 4, TMB_B_FULL = 8, TMB_B_EMPTY = 10, TMB_COLW_FULL = 12, TMB_COLW_EMPTY = 14, TMB_COUNT = 16 };

struct ThreshMmaArgs {
    const uint8_t* src;  // frames as given (cv_bridge encoding `enc`), device memory
    int enc, bpp;
    size_t row_stride, frame_stride;
    int use_tma;         // the tensor map describes src (3 bytes per pixel, strides multiples of 16)
    uint32_t* halo;
    int W, H, n_frames;
    int halo_tpr, halo_tiles_y;
    size_t halo_scale_stride, halo_frame_stride;
    int thresh_c;
    int tiles_x, tiles_y;  // CTA tiles (120 x 60 outputs) per frame
    StartRec* starts;
    Counters* counters;
    unsigned int max_starts;
    long long* prof;  // debugging: [gridDim.x][16 warps][TM_PROF_KINDS] wait cycles, or nullptr
};

// ---- PTX wrappers ------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t tm_smem(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void tm_mbar_init(uint64_t* b, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(tm_smem(b)), "r"(count) : "memory"); }
__device__ __forceinline__ void tm_mbar_wait(uint64_t* b, uint32_t parity) {
    uint32_t done;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(tm_smem(b)), "r"(parity) : "memory");
    } while (!done);
}
// optional wait-time accounting (ThreshMmaArgs::prof != nullptr): cycles every warp spends in each kind of wait
#define TM_PROF_KINDS 12
#define TM_WAIT(kind, barrier, parity)                 \
    do {                                               \
        if (PROF) {                                    \
            const long long t0_ = clock64();           \
            tm_mbar_wait(barrier, parity);             \
            prof_acc[kind] += clock64() - t0_;         \
        } else {                                       \
            tm_mbar_wait(barrier, parity);             \
        }                                              \
    } while (0)
__device__ __forceinline__ void tm_mbar_arrive(uint64_t* b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(tm_smem(b)) : "memory"); }
__device__ __forceinline__ void tm_mbar_expect_tx(uint64_t* b, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(tm_smem(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ uint64_t tm_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    // wgmma shared-memory matrix descriptor, K-major, no swizzle: start >> 4 [0,14), LBO >> 4 [16,30), SBO >> 4 [32,46),
    // base offset 0, layout type 0 (no swizzle) at [62,64)
    return (uint64_t)((saddr >> 4) & 0x3FFF) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) | ((uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32);
}
// D (64 x 112, s32) (+)= A (64 x 32, u8, shared) * B (112 x 32, u8, shared)^T, issued by a whole warpgroup.  Fragment: warp w of the
// warpgroup, lane l holds rows 16 w + l / 4 (+ 8) and columns 8 j + 2 (l % 4) (+ 1):  d[4 j + 2 h + e] = D[16 w + l / 4 + 8 h][8 j + 2 (l % 4) + e]
__device__ __forceinline__ void tm_wgmma(uint32_t (&d)[56], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %58, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n112k32.s32.u8.u8 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,"
        "%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55}, %56, %57, p;\n\t}"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]),
          "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]),
          "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]),
          "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]),
          "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void tm_wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void tm_wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void tm_wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accesses of the accumulator registers across wgmma issue / wait
__device__ __forceinline__ void tm_wg_fence_regs(uint32_t (&d)[56]) {
#pragma unroll
    for (int i = 0; i < 56; i++) asm volatile("" : "+r"(d[i])::"memory");
}
__device__ __forceinline__ void tm_fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// one lane of a converged warp (the same one every time); the single-thread TMA instructions are issued under it while the
// loop around them stays warp-uniform, so addresses live in uniform registers
__device__ __forceinline__ bool tm_elect() {
    uint32_t pred;
    asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
    return pred != 0;
}
template <int N>
__device__ __forceinline__ void tm_regs_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void tm_regs_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// 32x32 bit-matrix transpose across a warp: lane l holds row l (bit c = M[l][c]); on return lane l holds
// column l (bit r = M[r][l]).  Five butterfly steps (tests/hostsim checks the same code on the CPU).
__device__ __forceinline__ uint32_t warp_transpose32(uint32_t x, int lane) {
#pragma unroll
    for (int j = 16; j >= 1; j >>= 1) {
        const uint32_t m = j == 16 ? 0x0000FFFFu : (j == 8 ? 0x00FF00FFu : (j == 4 ? 0x0F0F0F0Fu : (j == 2 ? 0x33333333u : 0x55555555u)));
        const uint32_t p = __shfl_xor_sync(0xffffffffu, x, j);
        x = (lane & j) ? ((x & ~m) | ((p >> j) & m)) : ((x & m) | ((p & m) << j));
    }
    return x;
}

__device__ __forceinline__ void tm_tile_coords(const ThreshMmaArgs& a, int t, int* f, int* bx, int* by) {
    const int per = a.tiles_x * a.tiles_y;
    *f = t / per;
    const int rem = t - *f * per;
    *by = rem / a.tiles_x;
    *bx = rem - *by * a.tiles_x;
}
// The box starts on a 16-byte boundary of the row (TMA is only specified for 16-byte aligned boxes of this u32 view):
// 3 bytes per pixel -> the box starts `tm_box_lead` pixels left of the
// region, at a column that is a multiple of 16 (X0 - 28 = 120 bx - 28 = 8 bx + 4 mod 16).
__device__ __forceinline__ int tm_box_lead(int bx) { return (bx & 1) ? 12 : 4; }
// region of the tile lies inside the image: TMA (zero fill outside) may stage it
__device__ __forceinline__ bool tm_tile_interior(const ThreshMmaArgs& a, int bx, int by) {
    const int xs = bx * THR_OW - 28, ys = by * THR_OH - 26;
    return a.use_tma && xs - tm_box_lead(bx) >= 0 && xs + 180 <= a.W && ys >= 0 && ys + TM_N <= a.H;
}

// Four consecutive gray pixels of region row y (clamped), columns xs .. xs+3, straight from the frame in global memory.
__device__ __forceinline__ uint32_t tm_gray4_global(const ThreshMmaArgs& a, const uint8_t* frame, int y, int xs) {
    y = y < 0 ? 0 : (y > a.H - 1 ? a.H - 1 : y);
    const uint8_t* row = frame + (size_t)y * a.row_stride;
    uint32_t out = 0;
    if (a.enc == 2) {  // MONO8: BGR2GRAY of (g,g,g) is g
        if (xs >= 0 && xs + 3 < a.W && ((reinterpret_cast<uintptr_t>(row + xs) & 3) == 0)) return __ldg(reinterpret_cast<const uint32_t*>(row + xs));
#pragma unroll
        for (int k = 0; k < 4; k++) {
            int x = xs + k;
            x = x < 0 ? 0 : (x > a.W - 1 ? a.W - 1 : x);
            out |= (uint32_t)__ldg(row + x) << (8 * k);
        }
        return out;
    }
    const bool rgb = a.enc == 1;
    if (xs >= 0 && xs + 3 < a.W && ((reinterpret_cast<uintptr_t>(row + 3 * (size_t)xs) & 3) == 0)) {
        const uint32_t* p = reinterpret_cast<const uint32_t*>(row + 3 * (size_t)xs);
        const uint32_t w0 = __ldg(p), w1 = __ldg(p + 1), w2 = __ldg(p + 2);
        const uint32_t c0[4] = {w0 & 255u, w0 >> 24, (w1 >> 16) & 255u, (w2 >> 8) & 255u};
        const uint32_t c1[4] = {(w0 >> 8) & 255u, w1 & 255u, w1 >> 24, (w2 >> 16) & 255u};
        const uint32_t c2[4] = {(w0 >> 16) & 255u, (w1 >> 8) & 255u, w2 & 255u, w2 >> 24};
#pragma unroll
        for (int k = 0; k < 4; k++) out |= (rgb ? gray_of(c2[k], c1[k], c0[k]) : gray_of(c0[k], c1[k], c2[k])) << (8 * k);
        return out;
    }
#pragma unroll
    for (int k = 0; k < 4; k++) {
        int x = xs + k;
        x = x < 0 ? 0 : (x > a.W - 1 ? a.W - 1 : x);
        const uint32_t p0 = __ldg(row + 3 * (size_t)x), p1 = __ldg(row + 3 * (size_t)x + 1), p2 = __ldg(row + 3 * (size_t)x + 2);
        out |= (rgb ? gray_of(p2, p1, p0) : gray_of(p0, p1, p2)) << (8 * k);
    }
    return out;
}


// ---- start cracks in the column domain --------------------------------------------------------------
// Same exact prune rules as halo_row_starts (contour_walk.cuh), for a thread that holds COLUMN words: bit y of
// cm2..cp2 = pixel (x-2 .. x+2, y) of one 32-row band (= the 32 rows of a halo tile).  Pixel (x+dx, y-1) is
// (c_dx << 1), (x+dx, y+1) is (c_dx >> 1).  `col` is the column's index inside its halo tile (1..30 = interior);
// the rules that look two columns away only apply where that column is part of the tile word (halo_row_starts'
// 0xFFFFFFFC / 0x3FFFFFFF masks).  Only interior rows (bits 1..30) are reported.
__device__ __forceinline__ void halo_col_starts(uint32_t cm2, uint32_t cm1, uint32_t c0, uint32_t cp1, uint32_t cp2, int col, uint32_t* L, uint32_t* R) {
    const uint32_t up = c0 << 1, up_l = cm1 << 1, up_r = cp1 << 1;
    const uint32_t lone = c0 & ~(up | up_l | up_r | cm1 | cp1 | (c0 >> 1) | (cm1 >> 1) | (cp1 >> 1));
    uint32_t l = c0 & ~cm1 & ~(up & ~up_l) & ~lone;
    l &= ~(~up & ~up_l & up_r);
    if (col >= 2) l &= ~(up_l & ~cm2 & ~(cm2 << 1));
    uint32_t r = c0 & ~cp1 & ~(up & ~up_r) & ~lone;
    r &= ~(~up & ~up_r & up_l);
    if (col <= 29) r &= ~(up_r & ~cp2 & ~(cp2 << 1));
    *L = l & 0x7FFFFFFEu;
    *R = r & 0x7FFFFFFEu;
}

// Start-queue space in blocks of TM_START_BLOCK records per warp and side: one global atomic per block instead
// of one per halo tile (whose latency sat on the critical path of every tile).  Unused records of a block are
// written as FID_START_NULL, which the walk skips.
struct StartAlloc {
    unsigned int base, used;  // current block of this warp (records base .. base + TM_START_BLOCK), records handed out
};
__device__ __forceinline__ void start_fill_nulls(StartRec* starts, unsigned int max_starts, bool right, unsigned int from, unsigned int to, int lane) {
    const unsigned int cap = max_starts / 2;
    for (unsigned int i = from + lane; i < to; i += 32)
        if (i < cap) starts[right ? max_starts - 1 - i : i].v = FID_START_NULL;
}
// returns the queue position of the warp's first record (warp-uniform); n = records the warp needs (<= TM_START_BLOCK)
__device__ __forceinline__ unsigned int start_reserve(StartAlloc& al, unsigned int n, StartRec* starts, Counters* counters, unsigned int max_starts, bool right, int lane) {
    if (al.used + n > TM_START_BLOCK) {
        if (al.used < TM_START_BLOCK) start_fill_nulls(starts, max_starts, right, al.base + al.used, al.base + TM_START_BLOCK, lane);
        unsigned int b = 0;
        if (lane == 0) b = atomicAdd(&counters->n_starts[right ? 1 : 0], (unsigned int)TM_START_BLOCK);
        al.base = __shfl_sync(0xffffffffu, b, 0);
        al.used = 0;
    }
    const unsigned int pos = al.base + al.used;
    al.used += n;
    return pos;
}

// H_r of scale s for the warpgroup's 64 columns xm_lo .. xm_lo + 63 (region columns i = xm + 27 - r .. xm + 27 + r, r <= 25):
// k-steps 0..3 for xm_lo = 0, 2..5 for xm_lo = 64 cover that band for every scale (steps outside it add zeros), so the chain
// has a fixed length.  Asynchronous: tm_wg_wait0() before the accumulators are read.
__device__ __forceinline__ void tm_issue_scale(uint32_t (&acc)[56], uint64_t adesc0, uint64_t bdesc, int s, int xm_lo) {
    const int kk_lo = xm_lo >> 5;
    const uint64_t ad = adesc0 + (uint64_t)(s * (TM_A_BYTES >> 4)) + (uint64_t)(kk_lo * 32);
    const uint64_t bd = bdesc + (uint64_t)(kk_lo * (2 * TM_B_LBO >> 4));
    tm_wg_fence();
    tm_wg_fence_regs(acc);
#pragma unroll
    for (int k = 0; k < 4; k++) tm_wgmma(acc, ad + (uint64_t)(k * 32), bd + (uint64_t)(k * (2 * TM_B_LBO >> 4)), k > 0);
    tm_wg_commit();
    tm_wg_fence_regs(acc);
}
static_assert((0 + 63 + 27 + 25) >> 5 <= 3 && (64 + 27 - 25) >> 5 >= 2 && (64 + 63 + 27 + 25) >> 5 <= 5, "4 k-steps per warpgroup cover the widest band");

// ---------------------------------------------------------------------------------------------------
template <bool PROF>
__global__ void __launch_bounds__(TM_THREADS, 1) k_threshold_mma(const ThreshMmaArgs a, const __grid_constant__ CUtensorMap tmap) {
    extern __shared__ __align__(1024) uint8_t tm_smem_raw[];
    uint8_t* sA = tm_smem_raw + TM_OFF_A;
    uint8_t* sB = tm_smem_raw + TM_OFF_B;
    uint8_t* sStage = tm_smem_raw + TM_OFF_STAGE;
    uint32_t* sColw = reinterpret_cast<uint32_t*>(tm_smem_raw + TM_OFF_COLW);
    uint64_t* bar = reinterpret_cast<uint64_t*>(tm_smem_raw + TM_OFF_BAR);
    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);  // provably warp-uniform: the role branches stay convergent for wgmma
    const int total_tiles = a.tiles_x * a.tiles_y * a.n_frames;

    // ---- one-time setup: Hankel band tables, barriers ----
    for (int w = tid; w < TM_NTAB * TM_A_BYTES / 4; w += TM_THREADS) {
        const int tb = w / (TM_A_BYTES / 4), e = (w - tb * (TM_A_BYTES / 4)) * 4;
        const int r = 2 * tb + 1;
        const int d = e >> 7, row = (e >> 4) & 7, col = e & 15;
        uint32_t v = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            int s = 8 * d + row + col + k - TM_C0;
            s = s < 0 ? -s : s;
            v |= (s <= r ? 1u : 0u) << (8 * k);
        }
        reinterpret_cast<uint32_t*>(sA)[w] = v;
    }
    if (tid == 0) {
        for (int i = 0; i < TM_NSTAGES; i++) {
            tm_mbar_init(&bar[TMB_STAGE_FULL + i], 1);
            tm_mbar_init(&bar[TMB_STAGE_EMPTY + i], TM_NCONV);
        }
        for (int i = 0; i < 2; i++) {
            tm_mbar_init(&bar[TMB_B_FULL + i], TM_NCONV * 32);
            tm_mbar_init(&bar[TMB_B_EMPTY + i], TM_NEPI);
            tm_mbar_init(&bar[TMB_COLW_FULL + i], TM_NEPI);
            tm_mbar_init(&bar[TMB_COLW_EMPTY + i], TM_NCONV);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    tm_fence_async_smem();  // the band tables are read by the tensor core (async proxy)
    __syncthreads();
    long long prof_acc[PROF ? TM_PROF_KINDS : 1];
#pragma unroll
    for (int i = 0; i < (PROF ? TM_PROF_KINDS : 1); i++) prof_acc[i] = 0;
    const long long prof_t0 = PROF ? clock64() : 0;

    if (warp < TM_WARP_CONV0) {
      tm_regs_dec<TM_REGS_CTRL>();
      if (warp == TM_WARP_TMA) {
        // ===== TMA producer: BGR bands of the interior tiles into the stage ring (warp-uniform loop, one elected lane issues) =====
        uint32_t n_issued = 0;
        for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
            int f, bx, by;
            tm_tile_coords(a, t, &f, &bx, &by);
            if (!tm_tile_interior(a, bx, by)) continue;
            const int c0 = (3 * (bx * THR_OW - 28 - tm_box_lead(bx))) >> 2, c1 = by * THR_OH - 26;  // c0 is a multiple of 12: 16-byte aligned start
            for (int band = 0; band < TM_NBANDS; band++, n_issued++) {
                const uint32_t st = n_issued % TM_NSTAGES, use = n_issued / TM_NSTAGES;
                TM_WAIT(0, &bar[TMB_STAGE_EMPTY + st], (use & 1u) ^ 1u);
                if (tm_elect()) {
                    tm_mbar_expect_tx(&bar[TMB_STAGE_FULL + st], TM_STAGE_BYTES);
                    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(
                                     tm_smem(sStage + st * TM_STAGE_STRIDE)),
                                 "l"((uint64_t)&tmap), "r"(c0), "r"(c1 + band * TM_BOXH), "r"(f), "r"(tm_smem(&bar[TMB_STAGE_FULL + st]))
                                 : "memory");
                }
                __syncwarp();
            }
        }
      }  // warps 1-3: no role (they complete the first warpgroup so that setmaxnreg can hand its registers to the epilogue)
    } else if (warp < TM_WARP_EPI0) {
        // ===== converters: BGR -> gray into the MMA's B operand; then the halo tiles of the previous tile: the epilogue's
        //       column words (shared memory) -> 32x32 bit transposes -> one 128-byte store per tile and scale =====
        tm_regs_dec<TM_REGS_CONV>();
        const int cw = warp - TM_WARP_CONV0;
        const int nsub = lane >> 2, q = lane & 3;
        uint32_t n_consumed = 0;
        const int my_tiles = blockIdx.x < total_tiles ? (total_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
        for (int it = 0; it <= my_tiles; it++) {
            if (it < my_tiles) {
                const int t = blockIdx.x + it * gridDim.x;
                int f, bx, by;
                tm_tile_coords(a, t, &f, &bx, &by);
                const uint32_t buf = it & 1u, useb = (uint32_t)it >> 1;
                TM_WAIT(2, &bar[TMB_B_EMPTY + buf], (useb & 1u) ^ 1u);
                uint8_t* dstB = sB + buf * TM_B_BYTES;
                if (tm_tile_interior(a, bx, by)) {
                    const bool rgb = a.enc == 1;
                    const int woff = (3 * tm_box_lead(bx)) >> 2;  // the region starts 3 or 9 words into the staged row
                    for (int band = 0; band < TM_NBANDS; band++, n_consumed++) {
                        const uint32_t st = n_consumed % TM_NSTAGES, use = n_consumed / TM_NSTAGES;
                        TM_WAIT(1, &bar[TMB_STAGE_FULL + st], use & 1u);
                        const uint32_t* stage = reinterpret_cast<const uint32_t*>(sStage + st * TM_STAGE_STRIDE);
#pragma unroll 1
                        for (int blk = 0; blk < 6; blk++) {
                            const int b = cw + blk * TM_NCONV;       // 24 blocks of 8 rows x 16 columns per band
                            const int rg = b / 12, c = b - rg * 12;  // row group (0/1), column chunk
                            const int row = rg * 8 + nsub;
                            const uint32_t* p = stage + row * TM_BOXW + woff + 12 * c + 3 * q;
                            const uint32_t w0 = p[0], w1 = p[1], w2 = p[2];  // B0 G0 R0 B1 | G1 R1 B2 G2 | R2 B3 G3 R3
                            const uint32_t c0[4] = {w0 & 255u, w0 >> 24, (w1 >> 16) & 255u, (w2 >> 8) & 255u};
                            const uint32_t c1[4] = {(w0 >> 8) & 255u, w1 & 255u, w1 >> 24, (w2 >> 16) & 255u};
                            const uint32_t c2[4] = {(w0 >> 16) & 255u, (w1 >> 8) & 255u, w2 & 255u, w2 >> 24};
                            uint32_t g4 = 0;
#pragma unroll
                            for (int k = 0; k < 4; k++) g4 |= (rgb ? gray_of(c2[k], c1[k], c0[k]) : gray_of(c0[k], c1[k], c2[k])) << (8 * k);
                            *reinterpret_cast<uint32_t*>(dstB + c * TM_B_LBO + (band * TM_BOXH + row) * 16 + 4 * q) = g4;
                        }
                        __syncwarp();
                        if (lane == 0) tm_mbar_arrive(&bar[TMB_STAGE_EMPTY + st]);
                    }
                } else {
                    // replicate-border tile: clamping loads from global memory, three blocks (9 loads) in flight per thread
                    const uint8_t* frame = a.src + (size_t)f * a.frame_stride;
                    const int xs0 = bx * THR_OW - 28, ys0 = by * THR_OH - 26;
                    #pragma unroll 1
                    for (int b0 = cw; b0 < (TM_N / 8) * 12; b0 += 3 * TM_NCONV) {  // 168 blocks of 8 rows x 16 columns, 42 per warp
                        uint32_t g4[3];
#pragma unroll
                        for (int u = 0; u < 3; u++) {
                            const int b = b0 + u * TM_NCONV;
                            const int rg = b / 12, c = b - rg * 12;
                            g4[u] = b < (TM_N / 8) * 12 ? tm_gray4_global(a, frame, ys0 + rg * 8 + nsub, xs0 + 16 * c + 4 * q) : 0u;
                        }
#pragma unroll
                        for (int u = 0; u < 3; u++) {
                            const int b = b0 + u * TM_NCONV;
                            const int rg = b / 12, c = b - rg * 12;
                            if (b < (TM_N / 8) * 12) *reinterpret_cast<uint32_t*>(dstB + c * TM_B_LBO + (rg * 8 + nsub) * 16 + 4 * q) = g4[u];
                        }
                    }
                }
                tm_fence_async_smem();  // generic-proxy stores -> visible to the tensor core
                tm_mbar_arrive(&bar[TMB_B_FULL + buf]);
            }
            if (it > 0) {
                // halo tiles of tile it-1 (its epilogue runs while tile `it` was converted above)
                const int pt = blockIdx.x + (it - 1) * gridDim.x;
                int f, bx, by;
                tm_tile_coords(a, pt, &f, &bx, &by);
                const uint32_t pbuf = (uint32_t)(it - 1) & 1u, puse = (uint32_t)(it - 1) >> 1;
                const uint32_t* colw = sColw + pbuf * TM_COLW_WORDS;
                TM_WAIT(9, &bar[TMB_COLW_FULL + pbuf], puse & 1u);
                const int txl = cw;
                const int tx = bx * THR_TILES_X + txl;
#pragma unroll 1
                for (int tyl = 0; tyl < 2; tyl++) {
                    const int ty = by * THR_TILES_Y + tyl;
                    if (tx < a.halo_tpr && ty < a.halo_tiles_y) {
                        uint32_t* out = a.halo + (size_t)f * a.halo_frame_stride + ((size_t)ty * a.halo_tpr + tx) * 32 + lane;
#pragma unroll 1
                        for (int s = 0; s < 13; s++) out[(size_t)s * a.halo_scale_stride] = warp_transpose32(colw[(s * 2 + tyl) * 128 + FID_HALO_T * txl + lane], lane);
                    }
                }
                __syncwarp();
                if (lane == 0) tm_mbar_arrive(&bar[TMB_COLW_EMPTY + pbuf]);
            }
        }
    } else {
        // ===== MMA + epilogue: per scale one wgmma chain (64 columns x 112 region rows) into registers, parked in shared
        //       memory; vertical running sums, compare -> column words (shared memory) -> start cracks of the border walk =====
        tm_regs_inc<TM_REGS_EPI>();
        const int ew = warp - TM_WARP_EPI0;       // 0..7
        const int G = ew >> 2;                    // warpgroup: accumulator rows m = 64 G .. 64 G + 63 of the band matrix
        const int wq = ew & 3;                    // warp inside the warpgroup
        const int band = wq >> 1;                 // output rows 30 band .. 30 band + 31 (= halo tile row `band` of the tile)
        const int cl = ((wq & 1) << 5) | lane;    // this thread's column inside the warpgroup's 64
        const int xm = 127 - (64 * G + cl);       // column index within the tile's 122-column span (x = X0 - 1 + xm)
        const int y0 = 30 * band;
        const int xm_lo = G ? 0 : 64;             // columns of the warpgroup: xm_lo .. xm_lo + 63
        uint16_t* sD = reinterpret_cast<uint16_t*>(tm_smem_raw + TM_OFF_D + 2 * G * TM_D_BYTES);
        const uint64_t adesc0 = tm_desc(tm_smem(sA) + 1024u * (uint32_t)G, 256, 128);  // + table * (TM_A_BYTES >> 4) + kstep * 32
        const int twoC = 2 * a.thresh_c - 1;
        // this column inside its halo tile: xm = 1..120 are interior columns of tile (xm - 1) / 30 (local column 1..30)
        const int txl = xm >= 1 && xm <= 120 ? (xm - 1) / FID_HALO_T : -1;
        const int col = xm - FID_HALO_T * txl;
        StartAlloc alL{0u, (unsigned int)TM_START_BLOCK}, alR{0u, (unsigned int)TM_START_BLOCK};  // "block used up": the first reservation fetches one
        const unsigned int start_cap = a.max_starts / 2;
        bool start_overflow = false;
        uint32_t acc[56];
#pragma unroll
        for (int i = 0; i < 56; i++) acc[i] = 0;
        uint32_t it = 0;
        for (int t = blockIdx.x; t < total_tiles; t += gridDim.x, it++) {
            int f, bx, by;
            tm_tile_coords(a, t, &f, &bx, &by);
            const int X0 = bx * THR_OW, Y0 = by * THR_OH;
            const uint32_t buf = it & 1u, useb = it >> 1;
            uint32_t* colw = sColw + buf * TM_COLW_WORDS;
            TM_WAIT(8, &bar[TMB_COLW_EMPTY + buf], (useb & 1u) ^ 1u);  // the converter warps are done with this buffer (tile it - 2)
            // validity: bit b of the band's word <-> image row Y0 - 1 + y0 + b; column X0 - 1 + xm
            uint32_t rowmask;
            {
                const int lo = 1 - Y0 - y0, hi = a.H - Y0 - y0;  // valid b: lo <= b <= hi
                const uint32_t m_lo = lo <= 0 ? 0xffffffffu : (lo >= 32 ? 0u : (0xffffffffu << lo));
                const uint32_t m_hi = hi >= 31 ? 0xffffffffu : (hi < 0 ? 0u : (0xffffffffu >> (31 - hi)));
                rowmask = m_lo & m_hi;
            }
            const int X = X0 - 1 + xm;
            const bool col_ok = X >= 0 && X < a.W;
            TM_WAIT(3, &bar[TMB_B_FULL + buf], useb & 1u);
            const uint8_t* gB = sB + buf * TM_B_BYTES;
            // centre pixels of the band's 32 output rows (region rows 25 + y0 ..), region column xm + 27, straight from the gray tile
            uint32_t g4[8];
            {
                const int ic = xm + 27;
                const uint8_t* gp = gB + (ic >> 4) * TM_B_LBO + (25 + y0) * 16 + (ic & 15);
#pragma unroll
                for (int w = 0; w < 8; w++)
                    g4[w] = (uint32_t)gp[64 * w] | ((uint32_t)gp[64 * w + 16] << 8) | ((uint32_t)gp[64 * w + 32] << 16) | ((uint32_t)gp[64 * w + 48] << 24);
            }
            const uint64_t bdesc = tm_desc(tm_smem(gB), TM_B_LBO, 128);  // + kstep * (2 * TM_B_LBO >> 4)
            tm_issue_scale(acc, adesc0, bdesc, 0, xm_lo);
            for (int s = 0; s < 13; s++) {
                const uint32_t j = it * 13u + (uint32_t)s;  // global scale index: 13 is odd, so the parking buffers alternate across tiles too
                uint16_t* sDj = sD + (j & 1u) * (TM_D_BYTES / 2);
                tm_wg_wait0();
                tm_wg_fence_regs(acc);
                {  // park: H(column m, region row n) at sDj[m * TM_DSTRIDE + n], two rows per word
                    uint32_t* d32 = reinterpret_cast<uint32_t*>(sDj);
                    const int m0 = 16 * wq + (lane >> 2);
#pragma unroll
                    for (int jj = 0; jj < TM_N / 8; jj++)
#pragma unroll
                        for (int h = 0; h < 2; h++)
                            d32[(m0 + 8 * h) * (TM_DSTRIDE / 2) + 4 * jj + (lane & 3)] = (acc[4 * jj + 2 * h] & 0xffffu) | (acc[4 * jj + 2 * h + 1] << 16);
                }
                if (s == 12) {  // every MMA of this warp that reads the gray tile has completed, and its centre pixels are in registers
                    __syncwarp();
                    if (lane == 0) tm_mbar_arrive(&bar[TMB_B_EMPTY + buf]);
                }
                asm volatile("bar.sync %0, 128;" ::"r"(2 + G) : "memory");  // the warpgroup's parked scale is complete
                if (s < 12) tm_issue_scale(acc, adesc0, bdesc, s + 1, xm_lo);  // waited for at once (see the header)
                const int r = 1 + 2 * s, k = 2 * r + 1, k2 = k * k;
                const int ck = (twoC * k2 + 1) / 2;  // exact: odd * odd + 1 is even
                const int negk2 = -k2;
                const uint16_t* hc = sDj + cl * TM_DSTRIDE + y0;  // H(x, region row y0 + n)
                // V = sum of H over region rows y0 + 25 - r .. y0 + 25 + r (window of the band's first output row), minus the constant
                int V = -ck;
#pragma unroll 4
                for (int n = 25 - r; n <= 25 + r; n++) V += (int)hc[n];
                const uint16_t* lead = hc + 26 + r;
                const uint16_t* trail = hc + 25 - r;
                uint32_t w = 0;
#pragma unroll
                for (int i = 0; i < 32; i++) {
                    const int g = (int)((g4[i >> 2] >> (8 * (i & 3))) & 255u);
                    const int D = g * negk2 + V;  // S - g k^2 - ck: the pixel is set iff D >= 0
                    w |= (uint32_t)(D >= 0) << i;
                    if (i < 31) V += (int)lead[i] - (int)trail[i];
                }
                const uint32_t cwb = col_ok ? (w & rowmask) : 0u;
                colw[(s * 2 + band) * 128 + xm] = cwb;
                {
                    const long long t0_ = PROF ? clock64() : 0;
                    asm volatile("bar.sync 1, 256;" ::: "memory");  // all 128 column words of this scale are in shared memory
                    if (PROF) prof_acc[PROF ? 10 : 0] += clock64() - t0_;
                }
                // start cracks of this column, exact local prune; neighbour columns from shared memory
                uint32_t Lb = 0, Rb = 0;
                if (txl >= 0 && cwb) {
                    const uint32_t* cp = colw + (s * 2 + band) * 128 + xm;
                    halo_col_starts(xm >= 2 ? cp[-2] : 0u, cp[-1], cwb, cp[1], cp[2], col, &Lb, &Rb);
                }
                const unsigned int mine = (unsigned int)__popc(Lb) | ((unsigned int)__popc(Rb) << 16);  // both counts in one scan
                unsigned int incl = mine;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const unsigned int tv = __shfl_up_sync(0xffffffffu, incl, d);
                    if (lane >= d) incl += tv;
                }
                const unsigned int tot = __shfl_sync(0xffffffffu, incl, 31);
                if (tot == 0) continue;
                unsigned int pl = 0, pr = 0;
                if (tot & 0xffffu) pl = start_reserve(alL, tot & 0xffffu, a.starts, a.counters, a.max_starts, false, lane) + ((incl - mine) & 0xffffu);
                if (tot >> 16) pr = start_reserve(alR, tot >> 16, a.starts, a.counters, a.max_starts, true, lane) + ((incl - mine) >> 16);
                if (mine) {
                    const uint32_t tx = (uint32_t)(bx * THR_TILES_X + txl), ty = (uint32_t)(by * THR_TILES_Y + band);
                    const uint32_t rec = start_rec_pack((uint32_t)((f * a.halo_tiles_y + (int)ty) * a.halo_tpr + (int)tx), (uint32_t)s, 0u, (uint32_t)col);
                    while (Lb) {
                        const int row = __ffs(Lb) - 1;
                        Lb &= Lb - 1;
                        if (pl < start_cap)
                            a.starts[pl].v = rec | ((uint32_t)row << 5);
                        else
                            start_overflow = true;
                        pl++;
                    }
                    while (Rb) {
                        const int row = __ffs(Rb) - 1;
                        Rb &= Rb - 1;
                        if (pr < start_cap)
                            a.starts[a.max_starts - 1 - pr].v = rec | ((uint32_t)row << 5);
                        else
                            start_overflow = true;
                        pr++;
                    }
                }
            }
            __syncwarp();
            if (lane == 0) tm_mbar_arrive(&bar[TMB_COLW_FULL + buf]);  // this warp's column words of the tile are in shared memory
        }
        // hand the unused part of this warp's last blocks back as null records
        if (alL.used < TM_START_BLOCK) start_fill_nulls(a.starts, a.max_starts, false, alL.base + alL.used, alL.base + TM_START_BLOCK, lane);
        if (alR.used < TM_START_BLOCK) start_fill_nulls(a.starts, a.max_starts, true, alR.base + alR.used, alR.base + TM_START_BLOCK, lane);
        if (start_overflow) atomicOr(&a.counters->overflow, 1u);
    }
    if (PROF && lane == 0) {
        prof_acc[PROF ? 11 : 0] = clock64() - prof_t0;
        for (int i = 0; i < (PROF ? TM_PROF_KINDS : 1); i++) a.prof[((size_t)blockIdx.x * 16 + warp) * TM_PROF_KINDS + i] = prof_acc[i];
    }
}

}  // namespace fid
