// CUDA kernels, contour half of the per-frame pipeline (sm_90a); the threshold stage that feeds it
// is in kernels_threshold.cuh:
//   k_walk          one thread per start crack / suspended walk, in rounds: round 0 one-directional, later
//                   rounds bidirectional; canonical test, contour length, emission segments      (A.3b)
//   k_emit          one thread per contour segment: ordered contour points
//   k_approx_warp   one warp per contour (<= 1024 points): approxPolyDP + quad filters             (A.4)
//   k_approx        one block per longer contour
// All kernels take a batch of frames (blockIdx.z / queue entries carry the frame index) so that a
// launch has enough independent work to fill the 132 SMs of an H100.
#pragma once
#include <cuda_runtime.h>

#include "approx_quad.cuh"
#include "common.cuh"
#include "contour_walk.cuh"
#include "quad_group.cuh"

namespace fid {

// ---- batch-wide work queues ------------------------------------------------------------------------
#define FID_WALK_MAX_ROUNDS 8
struct Counters {
    unsigned int n_starts[2];  // left-crack / right-crack start queues
    unsigned int n_chains;
    unsigned int n_points;
    unsigned int overflow;  // bit0 starts, bit1 chains, bit2 points, bit3 raw quads, bit4 selected, bit5 markers, bit6 walk queue
    unsigned int n_q[FID_WALK_MAX_ROUNDS][2];  // walks suspended by each round, per direction
    unsigned int work[FID_WALK_MAX_ROUNDS][2]; // persistent-walker work counters, per direction
    unsigned int emit_work;
    unsigned int n_segs;       // contour segments queued for k_emit
    unsigned int approx_work;  // k_approx_warp work counter
    unsigned int n_first;      // selected candidates of the chunk (k_sort_group -> k_identify_first work list)
    unsigned int n_retry;      // candidates whose first identification attempt failed (-> k_identify_retry work list)
};

struct WalkRec {       // a bidirectional border walk suspended between rounds (contour_walk.cuh, WalkState2)
    uint32_t xy0;      // start pixel
    uint32_t meta;     // frame << 8 | scale << 1 | is_right
    uint32_t xyf;      // forward walker's pixel
    uint32_t xyb;      // backward walker's pixel
    uint32_t state;    // df | db << 3 | n << 6
    uint32_t nf;       // steps of the forward walker
};

// A start crack as the threshold kernel queues it: 4 bytes, relative to its halo tile.  The side (left /
// right crack) is the queue region it sits in.  [tile within the chunk : 18][scale : 4][tile row : 5][bit : 5]
struct StartRec {
    uint32_t v;
};
#define FID_START_TILE_BITS 18
#define FID_START_NULL 0xFFFFFFFFu  // padding of a partly used queue block (kernels_threshold_mma.cuh); tile field all ones never occurs
FID_HD uint32_t start_rec_pack(uint32_t tile, uint32_t scale, uint32_t row, uint32_t col) { return (tile << 14) | (scale << 10) | (row << 5) | col; }

struct ChainRec {
    uint32_t xy;
    uint32_t meta;
    uint32_t n;
    uint32_t offset;  // into the batch point buffer
};

struct FrameGeom {
    int W, H;
    int gray_pitch;     // bytes
    size_t bgr_row_stride, bgr_frame_stride;
    size_t gray_frame_stride;
    int halo_tpr, halo_tiles_y;  // 30x30(+halo) tiles per tile row / tile rows
    size_t halo_scale_stride, halo_frame_stride;  // in words (see HaloView)
    uint32_t magic_tpr, magic_tiles_y;  // ceil(2^32 / d): __umulhi(t, magic) == t / d for t < 2^18, d < 2^14
};

// start record -> (pixel, meta = frame << 8 | scale << 1 | is_right)
__device__ __forceinline__ void start_rec_unpack(const FrameGeom& g, uint32_t v, uint32_t is_right, uint32_t* xy, uint32_t* meta) {
    const uint32_t tile = v >> 14, scale = (v >> 10) & 15u, row = (v >> 5) & 31u, col = v & 31u;
    const uint32_t trow = __umulhi(tile, g.magic_tpr);            // f * tiles_y + ty
    const uint32_t tx = tile - trow * (uint32_t)g.halo_tpr;
    const uint32_t f = __umulhi(trow, g.magic_tiles_y);
    const uint32_t ty = trow - f * (uint32_t)g.halo_tiles_y;
    *xy = (FID_HALO_T * tx - 1u + col) | ((FID_HALO_T * ty - 1u + row) << 16);
    *meta = (f << 8) | (scale << 1) | is_right;
}

// ---------------------------------------------------------------------------------------------------
// Border walk in rounds of growing step budget.  Walk lengths are heavy tailed (most start cracks
// die within a few steps, a few percent walk hundreds, the canonical starts of marker outlines walk
// thousands) and the walk is issue bound, so idle lanes are the cost: each round walks every lane by
// at most its budget and re-queues the undecided walks, which keeps the lanes of a warp within one
// budget of each other; the last, long rounds run "persistent" (a lane that finishes pulls the next
// queue item when at least half the warp is idle).  Left-crack (backwards) and right-crack
// (forwards) walks live in separate queue regions, so a warp executes a single code path (the crack
// type decides the tie rule and, in round 0, the direction; rounds >= 1 walk both ways, contour_walk.cuh).
// ---------------------------------------------------------------------------------------------------
struct WalkArgs {
    const uint32_t* halo;
    const uint32_t* lut_prev;
    const uint32_t* lut_next;
    const StartRec* starts;   // round 0 input: left items at [0, nL), right items at [max_starts-1 ...]
    const WalkRec* q_in;      // later rounds: left items at [0, nL), right items at [max_queue-1 ...]
    WalkRec* q_out;
    ChainRec* chains;
    SegRec* segs;
    Counters* counters;
    unsigned int max_starts, max_chains, max_points, max_queue, max_segs;
    int round;                // 0 = items are start cracks
    FrameGeom g;
    int min_len, max_len, budget;
    int persistent;
    unsigned int chunk;       // persistent mode: queue items a warp takes per atomic
    int refill_min;           // persistent mode: refill the warp's idle lanes from the queue when at least this many are idle
    int pass_steps;           // persistent mode: steps every active lane walks between two refill checks
};

struct WalkItem {
    uint32_t xy0, meta;
    WalkState2 st;
    int x0, y0;
    WalkCtx ctx;
};

__device__ __forceinline__ WalkCtx walk_ctx_of(const WalkArgs& a, uint32_t meta) {
    const int f = meta >> 8, s = (meta >> 1) & 0x7F;
    WalkCtx ctx;
    ctx.plane = HaloView{a.halo + (size_t)f * a.g.halo_frame_stride + (size_t)s * a.g.halo_scale_stride, a.g.halo_tpr};
    ctx.lut_prev = a.lut_prev;
    ctx.lut_next = a.lut_next;
    return ctx;
}

template <bool IS_RIGHT>
__device__ __forceinline__ void walk_load_item(const WalkArgs& a, unsigned int idx, WalkItem& it) {
    const uint2* q = reinterpret_cast<const uint2*>(a.q_in + (IS_RIGHT ? a.max_queue - 1 - idx : idx));
    const uint2 w0 = q[0], w1 = q[1], w2 = q[2];
    it.xy0 = w0.x;
    it.meta = w0.y;
    it.st.xf = w1.x & 0xFFFF;
    it.st.yf = w1.x >> 16;
    it.st.xb = w1.y & 0xFFFF;
    it.st.yb = w1.y >> 16;
    it.st.df = w2.x & 7;
    it.st.db = (w2.x >> 3) & 7;
    it.st.n = w2.x >> 6;
    it.st.nf = w2.y;
    it.x0 = it.xy0 & 0xFFFF;
    it.y0 = it.xy0 >> 16;
    it.ctx = walk_ctx_of(a, it.meta);
}

template <bool IS_RIGHT>
__device__ __forceinline__ void walk_retire(const WalkArgs& a, int result, uint32_t xy0, uint32_t meta, const WalkState2& st, const WalkCtx& ctx, const WalkCkpt* ck) {
    if (result == WALK_CANONICAL && st.n >= a.min_len && st.n <= a.max_len) {
        const unsigned int slot = atomicAdd(&a.counters->n_chains, 1u);
        const unsigned int off = atomicAdd(&a.counters->n_points, ((unsigned int)st.n + 3u) & ~3u);  // 16-byte aligned chains
        if (slot < a.max_chains && off + (unsigned int)st.n <= a.max_points) {
            a.chains[slot] = ChainRec{xy0, meta, (uint32_t)st.n, off};
            const unsigned int nseg = (unsigned int)segment_count(ck);
            const unsigned int sbase = atomicAdd(&a.counters->n_segs, nseg);
            if (sbase + nseg <= a.max_segs) {
                SegRec* out = a.segs + sbase;
                make_segments(ctx, (int)(xy0 & 0xFFFF), (int)(xy0 >> 16), IS_RIGHT ? 1 : 0, st.n, st.nf, ck, meta, off,
                              [out](int k, const SegRec& sr) { *reinterpret_cast<uint4*>(out + k) = make_uint4(sr.xy, sr.meta, sr.dn, sr.off); });
            } else {
                a.chains[slot].n = 0;
                atomicOr(&a.counters->overflow, 2u);
            }
        } else {
            if (slot < a.max_chains) a.chains[slot] = ChainRec{xy0, meta, 0u, 0u};
            atomicOr(&a.counters->overflow, slot >= a.max_chains ? 2u : 4u);
        }
    } else if (result == WALK_CONTINUE) {
        const unsigned int pos = atomicAdd(&a.counters->n_q[a.round][IS_RIGHT ? 1 : 0], 1u);
        if (pos < a.max_queue / 2) {
            uint2* q = reinterpret_cast<uint2*>(a.q_out + (IS_RIGHT ? a.max_queue - 1 - pos : pos));
            q[0] = make_uint2(xy0, meta);
            q[1] = make_uint2((uint32_t)st.xf | ((uint32_t)st.yf << 16), (uint32_t)st.xb | ((uint32_t)st.yb << 16));
            q[2] = make_uint2((uint32_t)st.df | ((uint32_t)st.db << 3) | ((uint32_t)st.n << 6), (uint32_t)st.nf);
        } else {
            atomicOr(&a.counters->overflow, 64u);
        }
    }
}

template <bool IS_RIGHT>
__device__ __forceinline__ void walk_side(const WalkArgs& a, unsigned int n, unsigned int first_warp, unsigned int n_warps) {
    // `n` items of one direction, processed by warps first_warp .. first_warp+n_warps-1 of the grid
    const unsigned int lane = threadIdx.x & 31;
    const unsigned int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (warp < first_warp || warp >= first_warp + n_warps) return;
    const unsigned int my = warp - first_warp;
    if (a.round == 0) {
        // start cracks: one-directional walk "uphill" (left cracks backwards, right cracks forwards), which
        // disproves nine starts out of ten within the first few steps; survivors continue bidirectionally
        for (unsigned int base = my * 32; base < n; base += n_warps * 32) {
            const unsigned int idx = base + lane;
            if (idx >= n) continue;
            uint32_t sxy, smeta;
            const uint32_t srec = a.starts[IS_RIGHT ? a.max_starts - 1 - idx : idx].v;
            if (srec == FID_START_NULL) continue;
            start_rec_unpack(a.g, srec, IS_RIGHT ? 1u : 0u, &sxy, &smeta);
            const WalkCtx ctx = walk_ctx_of(a, smeta);
            const int x0 = sxy & 0xFFFF, y0 = sxy >> 16;
            WalkState st;
            if (walk_init(ctx, x0, y0, IS_RIGHT ? 1 : 0, &st) != WALK_CONTINUE) continue;
            const int r = walk_uni_fast<IS_RIGHT>(ctx, x0, y0, a.max_len, a.budget, &st);
            WalkState2 s2;
            walk_split<IS_RIGHT>(x0, y0, st, &s2);
            walk_retire<IS_RIGHT>(a, r, sxy, smeta, s2, ctx, nullptr);
        }
        return;
    }
    if (!a.persistent) {
        for (unsigned int base = my * 32; base < n; base += n_warps * 32) {
            const unsigned int idx = base + lane;
            if (idx >= n) continue;
            WalkItem it;
            walk_load_item<IS_RIGHT>(a, idx, it);
            const int r = walk_bidir_fast<IS_RIGHT>(it.ctx, it.x0, it.y0, a.max_len, a.budget, &it.st);
            walk_retire<IS_RIGHT>(a, r, it.xy0, it.meta, it.st, it.ctx, nullptr);
        }
        return;
    }
    // persistent lanes.  The first 32 * n_warps items are assigned statically, warp `my` taking items
    // [32 my, 32 my + 32): when there are fewer items than lanes (the long-walk rounds) the work is packed
    // into the lowest warps and every other warp -- and with it whole blocks and their registers -- retires
    // at once, leaving the SMs to whatever runs on the other streams.  Later items go through the counter.
    const unsigned int lt_mask = (1u << lane) - 1u;
    const unsigned int static_end = n_warps * 32u;
    unsigned int next = my * 32u, hi = next + 32u < n ? next + 32u : n;
    bool exhausted = false, active = false;
    if (next >= n) {
        if (static_end >= n) return;
        hi = next;  // nothing static for this warp; go to the counter
    }
    int budget_end = 0, last_f = 0, last_b = 0;
    WalkItem it;
    WalkCkpt ck;  // checkpoints of the current walk (local memory; touched once per FID_CKPT_STEP steps)
    ck.count[0] = ck.count[1] = 0;
    for (;;) {
        const uint32_t need = __ballot_sync(0xffffffffu, !active);
        if (__popc(need) >= a.refill_min) {  // refill when enough lanes are idle
            if (!exhausted && next >= hi) {
                unsigned int lo = 0;
                if (lane == 0) lo = atomicAdd(&a.counters->work[a.round][IS_RIGHT ? 1 : 0], a.chunk) + static_end;
                lo = __shfl_sync(0xffffffffu, lo, 0);
                next = lo;
                hi = lo + a.chunk < n ? lo + a.chunk : n;
                if (lo >= n) exhausted = true;
            }
            if (!exhausted) {
                const unsigned int want = (unsigned int)__popc(need);
                const unsigned int avail = hi - next;
                const unsigned int give = want < avail ? want : avail;
                const unsigned int rank = (unsigned int)__popc(need & lt_mask);
                if (!active && rank < give) {
                    walk_load_item<IS_RIGHT>(a, next + rank, it);
                    active = true;
                    budget_end = it.st.n + a.budget;
                    ck.count[0] = ck.count[1] = 0;
                    last_f = last_b = 0;
                }
                next += give;
            }
            if (exhausted && !__any_sync(0xffffffffu, active)) break;
        }
        if (active) {
            const int left = budget_end - it.st.n;
            const int r = walk_bidir_fast<IS_RIGHT>(it.ctx, it.x0, it.y0, a.max_len, left < a.pass_steps ? left : a.pass_steps, &it.st);
            if (r == WALK_CONTINUE && it.st.n < budget_end) {
                walk_checkpoint(it.st, &ck, &last_f, &last_b);
            } else {
                active = false;
                walk_retire<IS_RIGHT>(a, r, it.xy0, it.meta, it.st, it.ctx, &ck);
            }
        }
    }
}

__global__ void __launch_bounds__(256) k_walk(const WalkArgs a) {
    unsigned int nL, nR;
    if (a.round == 0) {
        nL = a.counters->n_starts[0];
        nR = a.counters->n_starts[1];
        const unsigned int cap = a.max_starts / 2;
        nL = nL < cap ? nL : cap;
        nR = nR < cap ? nR : cap;
    } else {
        nL = a.counters->n_q[a.round - 1][0];
        nR = a.counters->n_q[a.round - 1][1];
        const unsigned int cap = a.max_queue / 2;
        nL = nL < cap ? nL : cap;
        nR = nR < cap ? nR : cap;
    }
    // split the grid's warps between the two directions in proportion to their queue lengths
    const unsigned int total_warps = (gridDim.x * blockDim.x) >> 5;
    unsigned int wL = (unsigned int)(((unsigned long long)total_warps * nL) / ((unsigned long long)nL + nR + 1));
    if (nL && wL == 0) wL = 1;
    if (nR && wL >= total_warps) wL = total_warps - 1;
    if (!nR) wL = total_warps;
    if (nL) walk_side<false>(a, nL, 0, wL);
    if (nR) walk_side<true>(a, nR, wL, total_warps - wL);
}

// ---------------------------------------------------------------------------------------------------
// k_emit: one thread per surviving border writes its ordered points.
// ---------------------------------------------------------------------------------------------------
struct EmitArgs {
    const uint32_t* halo;
    const uint32_t* lut_prev;
    const uint32_t* lut_next;
    const SegRec* segs;
    Pt16* points;
    const Counters* counters;
    unsigned int* work_counter;
    unsigned int max_segs;
    FrameGeom g;
};

__global__ void __launch_bounds__(64) k_emit(const EmitArgs a) {
    // One thread per contour segment (contour_walk.cuh): at most ~FID_CKPT_STEP + one walk pass dependent
    // steps each.  Segments are handed out 32 at a time per warp through one atomic, from the END of
    // the list: the long-contour segments of the last walk round start first.
    unsigned int n = a.counters->n_segs;
    n = n < a.max_segs ? n : a.max_segs;
    const unsigned int lane = threadIdx.x & 31;
    for (;;) {
        unsigned int base = 0;
        if (lane == 0) base = atomicAdd(a.work_counter, 32u);
        base = __shfl_sync(0xffffffffu, base, 0);
        if (base >= n) break;
        const unsigned int k = base + lane;
        if (k < n) {
            const uint4 w = *reinterpret_cast<const uint4*>(a.segs + (n - 1 - k));
            const SegRec sr{w.x, w.y, w.z, w.w};
            const int f = sr.meta >> 8, s = (sr.meta >> 1) & 0x7F;
            const WalkCtx ctx{HaloView{a.halo + (size_t)f * a.g.halo_frame_stride + (size_t)s * a.g.halo_scale_stride, a.g.halo_tpr}, a.lut_prev, a.lut_next};
            trace_segment(ctx, sr, reinterpret_cast<uint32_t*>(a.points));
        }
        __syncwarp();
    }
}

// ---------------------------------------------------------------------------------------------------
// k_approx: one block per contour.
// ---------------------------------------------------------------------------------------------------
#define APPROX_THREADS 128
#define APPROX_WARP_MAX 1024  // contours up to this many points are handled by one warp (k_approx_warp)

struct BlockReducer {
    int* sh_val;  // [APPROX_THREADS/32]
    int* sh_idx;
    __device__ ArgMax reduce(int best_v, int best_j) const {
        // max value, ties -> smallest index (first maximum wins)
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
            const int ov = __shfl_xor_sync(0xffffffffu, best_v, d);
            const int oj = __shfl_xor_sync(0xffffffffu, best_j, d);
            if (ov > best_v || (ov == best_v && oj < best_j)) {
                best_v = ov;
                best_j = oj;
            }
        }
        const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        __syncthreads();  // protect sh_* from the previous call
        if (lane == 0) {
            sh_val[warp] = best_v;
            sh_idx[warp] = best_j;
        }
        __syncthreads();
        ArgMax r = {sh_val[0], sh_idx[0]};
#pragma unroll
        for (int w = 1; w < APPROX_THREADS / 32; w++) {
            const int ov = sh_val[w], oj = sh_idx[w];
            if (ov > r.value || (ov == r.value && oj < r.index)) {
                r.value = ov;
                r.index = oj;
            }
        }
        if (r.value == 0) r.index = 0;
        return r;
    }
    __device__ ArgMax farthest(const Pt16* p, int n, int pos0, int len) const {
        const int sx = p[pos0].x, sy = p[pos0].y;
        int bv = 0, bj = 0x7fffffff;
        for (int j = 1 + threadIdx.x; j < len; j += APPROX_THREADS) {
            int pos = pos0 + j;
            pos = pos >= n ? pos - n : pos;
            const Pt16 q = p[pos];
            const int dx = q.x - sx, dy = q.y - sy;
            const int d = dx * dx + dy * dy;
            if (d > bv) {
                bv = d;
                bj = j;
            }
        }
        return reduce(bv, bj);
    }
    __device__ ArgMax off_chord(const Pt16* p, int n, int s0, int s1) const {
        const int sx = p[s0].x, sy = p[s0].y;
        const int dx = p[s1].x - sx, dy = p[s1].y - sy;
        int len = s1 - s0;
        len = len <= 0 ? len + n : len;  // interior points are j = 1 .. len-1
        int bv = 0, bj = 0x7fffffff;
        for (int j = 1 + threadIdx.x; j < len; j += APPROX_THREADS) {
            int pos = s0 + j;
            pos = pos >= n ? pos - n : pos;
            const Pt16 q = p[pos];
            int d = (q.y - sy) * dx - (q.x - sx) * dy;
            d = d < 0 ? -d : d;
            if (d > bv) {
                bv = d;
                bj = j;
            }
        }
        return reduce(bv, bj);
    }
};

struct ApproxArgs {
    const ChainRec* chains;
    const Pt16* points;
    const Counters* counters;
    RawQuad* raw;           // [n_frames][max_raw]
    unsigned int* n_raw;    // [n_frames]
    Counters* counters_rw;
    unsigned int max_chains;
    int max_raw;
    int W, H;
    double poly_accuracy_rate, min_corner_dist_rate;
};

__device__ __forceinline__ void approx_emit_quad(const ApproxArgs& a, const ChainRec& c, const Pt16* q) {
    if (!quad_passes_filters(q, (int)c.n, a.W, a.H, a.min_corner_dist_rate)) return;
    const int f = c.meta >> 8, s = (c.meta >> 1) & 0x7F, is_right = c.meta & 1;
    const unsigned int slot = atomicAdd(&a.n_raw[f], 1u);
    if (slot < (unsigned int)a.max_raw) {
        RawQuad r;
        for (int k = 0; k < 4; k++) {
            r.x[k] = q[k].x;
            r.y[k] = q[k].y;
        }
        r.n_contour = (int)c.n;
        r.pts_off = c.offset;
        r.order_hi = (uint32_t)s;
        const uint32_t x = c.xy & 0xFFFF, y = c.xy >> 16;
        r.order_lo = 0xFFFFFFFFu - ((y * (uint32_t)a.W + x) * 2u + (uint32_t)is_right);
        a.raw[(size_t)f * a.max_raw + slot] = r;
    } else {
        atomicOr(&a.counters_rw->overflow, 8u);
    }
}

// Contours longer than APPROX_WARP_MAX points: one block per contour.
__global__ void __launch_bounds__(APPROX_THREADS) k_approx(const ApproxArgs a) {
    __shared__ int sh_val[APPROX_THREADS / 32], sh_idx[APPROX_THREADS / 32];
    unsigned int n = a.counters->n_chains;
    n = n < a.max_chains ? n : a.max_chains;
    BlockReducer red{sh_val, sh_idx};
    for (unsigned int i = blockIdx.x; i < n; i += gridDim.x) {
        const ChainRec c = a.chains[n - 1 - i];  // the long contours are at the end of the list
        if (c.n <= APPROX_WARP_MAX) continue;
        const Pt16* p = a.points + c.offset;
        Pt16 q[FID_APPROX_MAX_V];
        const int nv = approx_poly_closed(red, p, (int)c.n, (double)c.n * a.poly_accuracy_rate, q);
        if (nv != 4) continue;
        if (threadIdx.x == 0) approx_emit_quad(a, c, q);
    }
}

// Contours of at most APPROX_WARP_MAX points (nearly all of them): one WARP per contour, the points staged
// once in shared memory, every arg-max sweep a shuffle reduction -- no block barrier, no re-read from L2.
// (One block per contour spent ~190 instructions per point and sweep on a 100-point contour, nearly all of
// it in the block reduction.)
struct WarpReducer {
    __device__ ArgMax reduce(int best_v, int best_j) const {
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
            const int ov = __shfl_xor_sync(0xffffffffu, best_v, d);
            const int oj = __shfl_xor_sync(0xffffffffu, best_j, d);
            if (ov > best_v || (ov == best_v && oj < best_j)) {
                best_v = ov;
                best_j = oj;
            }
        }
        ArgMax r = {best_v, best_j};
        if (r.value == 0) r.index = 0;
        return r;
    }
    __device__ ArgMax farthest(const Pt16* p, int n, int pos0, int len) const {
        const int sx = p[pos0].x, sy = p[pos0].y;
        int bv = 0, bj = 0x7fffffff;
        for (int j = 1 + (int)(threadIdx.x & 31); j < len; j += 32) {
            int pos = pos0 + j;
            pos = pos >= n ? pos - n : pos;
            const Pt16 q = p[pos];
            const int dx = q.x - sx, dy = q.y - sy;
            const int d = dx * dx + dy * dy;
            if (d > bv) {
                bv = d;
                bj = j;
            }
        }
        return reduce(bv, bj);
    }
    __device__ ArgMax off_chord(const Pt16* p, int n, int s0, int s1) const {
        const int sx = p[s0].x, sy = p[s0].y;
        const int dx = p[s1].x - sx, dy = p[s1].y - sy;
        int len = s1 - s0;
        len = len <= 0 ? len + n : len;  // interior points are j = 1 .. len-1
        int bv = 0, bj = 0x7fffffff;
        for (int j = 1 + (int)(threadIdx.x & 31); j < len; j += 32) {
            int pos = s0 + j;
            pos = pos >= n ? pos - n : pos;
            const Pt16 q = p[pos];
            int d = (q.y - sy) * dx - (q.x - sx) * dy;
            d = d < 0 ? -d : d;
            if (d > bv) {
                bv = d;
                bj = j;
            }
        }
        return reduce(bv, bj);
    }
};

__global__ void __launch_bounds__(APPROX_THREADS) k_approx_warp(const ApproxArgs a) {
    __shared__ uint32_t sh_pts[APPROX_THREADS / 32][APPROX_WARP_MAX];
    unsigned int n = a.counters->n_chains;
    n = n < a.max_chains ? n : a.max_chains;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint32_t* mine = sh_pts[warp];
    const WarpReducer red;
    for (;;) {
        unsigned int i = 0;
        if (lane == 0) i = atomicAdd(&a.counters_rw->approx_work, 1u);
        i = __shfl_sync(0xffffffffu, i, 0);
        if (i >= n) break;
        const ChainRec c = a.chains[i];
        if (c.n == 0 || c.n > APPROX_WARP_MAX) continue;
        const uint32_t* src = reinterpret_cast<const uint32_t*>(a.points + c.offset);  // chains are 16-byte aligned
        const int n4 = ((int)c.n + 3) >> 2;
        for (int k = lane; k < n4; k += 32) reinterpret_cast<uint4*>(mine)[k] = reinterpret_cast<const uint4*>(src)[k];
        __syncwarp();
        Pt16 q[FID_APPROX_MAX_V];
        const int nv = approx_poly_closed(red, reinterpret_cast<const Pt16*>(mine), (int)c.n, (double)c.n * a.poly_accuracy_rate, q);
        if (nv == 4 && lane == 0) approx_emit_quad(a, c, q);
        __syncwarp();
    }
}

}  // namespace fid
