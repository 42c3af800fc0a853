// CUDA kernels, back half of the per-frame pipeline (sm_90a):
//   k_sort_group  one block per frame: clockwise fix, stable descending-perimeter order, pairwise
//                 "too close" matrix, OpenCV's order-dependent grouping                  (SURVEY A.5)
//   k_identify_first / k_identify_retry   one warp per selected candidate, one block per failed first attempt: perspective removal, Otsu, cell votes, border
//                 check, first-match dictionary search (+ close-contour retry)           (A.6, A.7)
//   k_finish      one block per frame: compaction in OpenCV's output order, cornerSubPix (A.8),
//                 solvePnP(ITERATIVE) + FiducialTransform arithmetic                     (A.9)
//   k_pose_hypotheses  opt-in, after k_finish: both IPPE_SQUARE solutions per marker (ippe.cuh)
//   k_board_pose  opt-in, after k_finish (and k_pose_hypotheses): one warp per (frame, board), one solvePnP over every
//                 detected marker of the board (board_pnp.cuh)
//   k_charuco     opt-in, last: one block per (frame, ChArUco board), its chessboard corners and pose (charuco.cuh)
//   k_marker_refine  one block per frame: board markers recovered from the rejected candidates (marker_refine.cuh)
//   k_rejected    opt-in, after k_finish: one block per frame, detectMarkers' rejected list (candidate_tree.cuh)
//   k_recovered_pose  opt-in, after k_marker_refine in a batch: the poses of the recovered markers
//   k_diamond     opt-in, last: one block per frame, its ChArUco diamonds and their poses (diamond.cuh)
#pragma once
#include <cuda_runtime.h>

#include "../../include/fiducials_b200.h"
#include "aruco3.cuh"
#include "board_pnp.cuh"
#include "candidate_tree.cuh"
#include "charuco.cuh"
#include "common.cuh"
#include "contour_refine.cuh"
#include "diamond.cuh"
#include "identify.cuh"
#include "ippe.cuh"
#include "marker_refine.cuh"
#include "pnp.cuh"
#include "quad_group.cuh"
#include "subpix.cuh"

namespace fid {

// The active dictionary lives in global memory as n_markers x 4 rotations of 64-bit words (params_host.h, pack_dictionary;
// any OpenCV predefined dictionary, up to 2320 markers x 32 B = 74 KB -- more than constant memory holds) and is staged into
// shared memory by every identification block.

struct FrameScratch {     // per-frame global scratch, all arrays sized max_raw
    QuadF* quads_tmp;     // clockwise quads, unsorted
    float* per_tmp;
    QuadF* quads;         // sorted
    float* per;           // sorted
    uint32_t* close_bits; // max_raw x close_wpr
    int* group_id;
    int* group_members;
    int* next_in_group;
    int* group_head;
    int* group_tail;
    int* close_count;
    int* close_idx;
    int* close_off;
    uint8_t* selected;
    int* sel_idx;         // selected candidates (sorted indices), in order
    int* raw_of_sorted;   // sorted index -> index into the frame's raw candidate list (its contour: CORNER_REFINE_CONTOUR)
};

struct GroupArgs {
    const RawQuad* raw;          // [F][max_raw]
    const unsigned int* n_raw;   // [F]
    FrameScratch fs;             // base pointers; frame f uses offset f*max_raw (close_bits: f*max_raw*close_wpr)
    int* n_sel;                  // [F]
    int* n_raw_clamped;          // [F]
    int max_raw, close_wpr, max_sel;
    int marker_size, border_bits;
    float min_marker_dist_rate, min_group_dist;
    int W, H, min_dist_to_border;
    Counters* counters;
    uint32_t* first_list;  // [F * max_sel] frame << 16 | k of every selected candidate of the chunk, any order
    int prof;  // FID_GROUP_PROF=1: frame 0 prints its phase clocks (debug aid)
};

// One warp as a lane group (identify.cuh, quad_group.cuh); tests/hostsim plugs SerialLanes (one lane).
struct WarpLanes {
    __device__ int lane() const { return threadIdx.x & 31; }
    __device__ int count() const { return 32; }
    __device__ void sync() const { __syncwarp(); }
    __device__ long long sum(long long v) const {
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
        return v;
    }
    __device__ int min_i(int v) const {
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
            const int o = __shfl_xor_sync(0xffffffffu, v, d);
            v = o < v ? o : v;
        }
        return v;
    }
    __device__ unsigned long long or_u64(unsigned long long v) const {
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) v |= __shfl_xor_sync(0xffffffffu, v, d);
        return v;
    }
    __device__ void hist_add(int* h, int bin) const { atomicAdd(h + bin, 1); }
    __device__ uint32_t ballot(bool p) const { return __ballot_sync(0xffffffffu, p); }
    __device__ int shfl_i(int v, int src) const { return __shfl_sync(0xffffffffu, v, src); }
    __device__ int atomic_add(int* p, int v) const { return atomicAdd(p, v); }
};

#define GROUP_THREADS 1024
#define FID_GROUP_MAX_RAW 4096  // >= fid_detector::max_raw
#define GROUP_CLOSE_SMEM_WORDS 12288  // 48 KB of the close-pair matrix in shared memory

// INV (detectInvertedMarker, DESIGN.md finding 18 B): every group keeps its smallest member (group_finish_lanes<true>).
template <bool INV = false>
__global__ void __launch_bounds__(GROUP_THREADS) k_sort_group(const GroupArgs a) {
    const int f = blockIdx.x;
    const int tid = threadIdx.x;
    int n = (int)a.n_raw[f];
    n = n < a.max_raw ? n : a.max_raw;
    const size_t fo = (size_t)f * a.max_raw;
    const RawQuad* raw = a.raw + fo;
    QuadF* qt = a.fs.quads_tmp + fo;
    float* pt = a.fs.per_tmp + fo;
    QuadF* qs = a.fs.quads + fo;
    float* ps = a.fs.per + fo;
    long long t_[7] = {0, 0, 0, 0, 0, 0, 0};
#define GROUP_TICK(k) if (a.prof && tid == 0 && f == 0) t_[k] = clock64()
    GROUP_TICK(0);
    if (tid == 0) a.n_raw_clamped[f] = n;
    extern __shared__ int sm_group[];  // 6 * max_raw ints + max_raw bytes (+ the close-pair matrix when it fits)
    // the grouping scratch is idle until pass 1: phases a-c keep their per-candidate scalars there (perimeters for the rank
    // sort, then centroids and distance thresholds for the close-pair pre-filter) instead of re-reading them from L2 in the
    // inner loops
    float* s_f0 = reinterpret_cast<float*>(sm_group);
    float* s_f1 = s_f0 + a.max_raw;
    float* s_f2 = s_f1 + a.max_raw;
    // a. clockwise + perimeter
    for (int i = tid; i < n; i += GROUP_THREADS) {
        const QuadF q = quad_clockwise(raw[i]);
        qt[i] = q;
        const float p = quad_perimeter(q);
        pt[i] = p;
        s_f0[i] = p;
    }
    __syncthreads();
    // b. rank = position under std::stable_sort(descending perimeter) of OpenCV's candidate order
    for (int i = tid; i < n; i += GROUP_THREADS) {
        const float pi = s_f0[i];
        const uint32_t hi = raw[i].order_hi, lo = raw[i].order_lo;
        int rank = 0;
        for (int j = 0; j < n; j++) {
            const float pj = s_f0[j];
            const bool before = pj > pi || (pj == pi && (raw[j].order_hi < hi || (raw[j].order_hi == hi && raw[j].order_lo < lo)));
            rank += before ? 1 : 0;
        }
        qs[rank] = qt[i];
        ps[rank] = pi;
        a.fs.raw_of_sorted[fo + rank] = i;
    }
    __syncthreads();
    QuadF* s_quads = reinterpret_cast<QuadF*>(s_f2 + a.max_raw);  // the other half of the scratch: up to 3 * max_raw / 8 quads
    const bool quads_in_smem = (size_t)n * sizeof(QuadF) <= (size_t)3 * a.max_raw * sizeof(int);
    for (int i = tid; i < n; i += GROUP_THREADS) {  // sorted order: centroid and "too close" threshold of every candidate
        const QuadF q = qs[i];
        s_f0[i] = (q.x[0] + q.x[1] + q.x[2] + q.x[3]) * 0.25f;
        s_f1[i] = (q.y[0] + q.y[1] + q.y[2] + q.y[3]) * 0.25f;
        s_f2[i] = ps[i] * a.min_marker_dist_rate;
        if (quads_in_smem) s_quads[i] = q;
    }
    __syncthreads();
    GROUP_TICK(1);
    // c. close-pair matrix, upper triangle; unit = (row i, 32-column word).  The matrix is very sparse (a
    //    marker scene has a few dozen close pairs among ~10^5): rows with at least one pair are flagged in
    //    shared memory so that the serial pass below does not pay an L2 round trip per empty word.
    __shared__ uint32_t row_any[(FID_GROUP_MAX_RAW + 31) / 32], grouped[(FID_GROUP_MAX_RAW + 31) / 32];
    int* sm_group_id = sm_group;
    int* sm_members = sm_group + a.max_raw;  // 2 * max_raw: members + accepted ids of every group
    int* sm_next = sm_group + 3 * a.max_raw;
    int* sm_head = sm_group + 4 * a.max_raw;
    int* sm_tail = sm_group + 5 * a.max_raw;
    uint8_t* sm_selected = reinterpret_cast<uint8_t*>(sm_group + 6 * a.max_raw);
    __shared__ int s_warp_cnt[GROUP_THREADS / 32];
    __shared__ int s_base;
    for (int i = tid; i < (FID_GROUP_MAX_RAW + 31) / 32; i += GROUP_THREADS) row_any[i] = 0;
    __syncthreads();
    const int wpr = (n + 31) >> 5;
    // the matrix lives in shared memory when it fits (n <= ~600 candidates): the serial pass below reads it
    // word by word, each read feeding the next decision -- from global memory that was an L2 round trip
    // per word and 2/3 of this kernel's time
    uint32_t* sm_close = reinterpret_cast<uint32_t*>(sm_selected + ((a.max_raw + 15) & ~15));
    const bool close_in_smem = n * wpr <= GROUP_CLOSE_SMEM_WORDS;
    uint32_t* cb = close_in_smem ? sm_close : a.fs.close_bits + fo * a.close_wpr;
    const int cb_pitch = close_in_smem ? wpr : a.close_wpr;
    // one warp per (row i, word w): lane = column j0 + lane, the word is a ballot.  The pre-filter -- the mean squared corner
    // distance is >= the squared centroid distance for every corner alignment, so a far centroid can never be "close"
    // (conservative margin) -- runs on shared memory; only the few near pairs load the two quads.
    {
        const int warp = tid >> 5, lane = tid & 31;
        for (int u = warp; u < n * wpr; u += GROUP_THREADS / 32) {
            const int i = u / wpr, w = u - i * wpr;
            const int j0 = w << 5;
            uint32_t bits = 0;
            if (j0 + 31 > i) {
                const int j = j0 + lane;
                bool close = false;
                if (j > i && j < n) {
                    const float thr = s_f2[j];
                    const float dx = s_f0[i] - s_f0[j], dy = s_f1[i] - s_f1[j];
                    const float cd2 = dx * dx + dy * dy;
                    const float lim = thr * 1.01f + 1.0f;
                    if (cd2 <= lim * lim) close = (quads_in_smem ? quad_avg_distance(s_quads[i], s_quads[j]) : quad_avg_distance(qs[i], qs[j])) < thr;
                }
                bits = __ballot_sync(0xffffffffu, close);
            }
            if (lane == 0) {
                cb[(size_t)i * cb_pitch + w] = bits;
                if (bits) atomicOr(&row_any[i >> 5], 1u << (i & 31));
            }
        }
    }
    __syncthreads();
    GROUP_TICK(2);
    // d. order-dependent grouping.  Pass 1 (the close pairs in row-major order -> groups) is inherently serial
    //    and runs in one thread on shared-memory scratch; pass 2 (per group: sort, pick the leader, collect the
    //    close contours that differ from the running reference) runs one warp per group.
    __shared__ int s_n_groups, s_total_close, s_members_used;
    __shared__ uint32_t s_row[2][FID_GROUP_MAX_RAW / 32], s_rowmask[2][4];
    if (tid < 32) {
        // warp 0: the lanes stage row i of the matrix (one coalesced load, the next row's load already in flight), lane 0
        // applies the sequential rule from shared memory.  A large frame (C4: ~1400 candidates, matrix in global memory) used
        // to pay one dependent L2 round trip per word of every row -- 20 ms per 4K frame.
        struct RowPtr {
            const uint32_t* p;
            __device__ uint32_t operator()(int w) const { return p[w]; }
        };
        const int lane = tid;
        int n_groups = 0;
        if (lane == 0) group_pairs_init(n, sm_selected, sm_group_id, sm_next, a.fs.close_count + fo, grouped);
        __syncwarp();
        auto next_row = [&](int i) {  // first row >= i with a close pair (warp uniform)
            while (i < n && !((row_any[i >> 5] >> (i & 31)) & 1u)) i++;
            return i;
        };
        if (close_in_smem) {
            if (lane == 0)
                for (int i = next_row(0); i < n; i = next_row(i + 1))
                    group_pairs_row(n, i, RowPtr{sm_close + (size_t)i * wpr}, nullptr, &n_groups, sm_selected, sm_group_id, sm_next, sm_head, sm_tail, grouped);
        } else {
            // three rows in flight: the L2 latency of a row hides behind the sequential work on the rows before it
            uint32_t v[3][4];
            int rows[3];
            rows[0] = next_row(0);
            rows[1] = rows[0] < n ? next_row(rows[0] + 1) : n;
            rows[2] = rows[1] < n ? next_row(rows[1] + 1) : n;
#pragma unroll
            for (int r = 0; r < 3; r++)
#pragma unroll
                for (int k = 0; k < 4; k++) v[r][k] = (rows[r] < n && lane + 32 * k < wpr) ? cb[(size_t)rows[r] * cb_pitch + lane + 32 * k] : 0u;
            int buf = 0;
            while (rows[0] < n) {
                const int i = rows[0];
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    if (lane + 32 * k < wpr) s_row[buf][lane + 32 * k] = v[0][k];
                    const uint32_t nz = __ballot_sync(0xffffffffu, v[0][k] != 0u);
                    if (lane == 0) s_rowmask[buf][k] = nz;
                }
                __syncwarp();
                const int inext = rows[2] < n ? next_row(rows[2] + 1) : n;
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    v[0][k] = v[1][k];
                    v[1][k] = v[2][k];
                    v[2][k] = (inext < n && lane + 32 * k < wpr) ? cb[(size_t)inext * cb_pitch + lane + 32 * k] : 0u;
                }
                rows[0] = rows[1];
                rows[1] = rows[2];
                rows[2] = inext;
                if (lane == 0) group_pairs_row(n, i, RowPtr{s_row[buf]}, s_rowmask[buf], &n_groups, sm_selected, sm_group_id, sm_next, sm_head, sm_tail, grouped);
                __syncwarp();
                buf ^= 1;
            }
        }
        if (lane == 0) {
            s_n_groups = n_groups;
            s_total_close = 0;
            s_members_used = 0;
            s_base = 0;
        }
    }
    __syncthreads();
    GROUP_TICK(3);
    {
        const WarpLanes L;
        for (int g = tid >> 5; g < s_n_groups; g += GROUP_THREADS / 32)
            group_finish_lanes<INV>(L, g, qs, a.marker_size, a.border_bits, a.min_group_dist, sm_selected, sm_members, &s_members_used, sm_next, sm_head, a.fs.close_count + fo,
                               a.fs.close_idx + fo, a.fs.close_off + fo, &s_total_close);
    }
    __syncthreads();
    GROUP_TICK(4);
    // e. selected candidates, in order, minus the ones near the frame border (dropped silently, with their group)
    for (int c0 = 0; c0 < n; c0 += GROUP_THREADS) {
        const int i = c0 + tid;
        const bool keep = i < n && sm_selected[i] && !quad_near_border(qs[i], a.W, a.H, a.min_dist_to_border);
        const uint32_t m = __ballot_sync(0xffffffffu, keep);
        const int lane = tid & 31, warp = tid >> 5;
        if (lane == 0) s_warp_cnt[warp] = __popc(m);
        __syncthreads();
        int off = s_base;
        for (int w = 0; w < warp; w++) off += s_warp_cnt[w];
        if (keep) {
            const int pos = off + __popc(m & ((1u << lane) - 1u));
            if (pos < a.max_sel)
                a.fs.sel_idx[fo + pos] = i;
            else
                atomicOr(&a.counters->overflow, 16u);
        }
        __syncthreads();
        if (tid == 0) {
            int tot = 0;
            for (int w = 0; w < GROUP_THREADS / 32; w++) tot += s_warp_cnt[w];
            s_base += tot;
        }
        __syncthreads();
    }
    {
        const int ns = s_base < a.max_sel ? s_base : a.max_sel;
        __shared__ unsigned int s_first_base;
        if (tid == 0) {
            a.n_sel[f] = ns;
            s_first_base = ns ? atomicAdd(&a.counters->n_first, (unsigned int)ns) : 0u;
        }
        __syncthreads();
        for (int j = tid; j < ns; j += GROUP_THREADS) a.first_list[s_first_base + j] = ((uint32_t)f << 16) | (uint32_t)j;
    }
    GROUP_TICK(5);
    if (a.prof && tid == 0 && f == 0)
        printf("[group prof] n=%d groups=%d clocks: sort %lld close %lld pass1 %lld pass2 %lld select %lld\n", n, s_n_groups, t_[1] - t_[0], t_[2] - t_[1], t_[3] - t_[2], t_[4] - t_[3], t_[5] - t_[4]);
#undef GROUP_TICK
}

// ---------------------------------------------------------------------------------------------------

struct IdentifyArgs {
    const uint8_t* src;  // the frames as given (encoding enc): gray is computed per sample, no gray plane
    size_t row_stride, frame_stride;
    int enc, W, H;
    FrameScratch fs;
    const int* n_sel;
    int max_raw;
    int max_sel;
    DevParams P;
    const unsigned long long* dict;  // n_markers * 4 words
    int* cand_id;        // [F][max_sel]  -1 rejected
    float* cand_corners; // [F][max_sel][8] rotated to marker order
    int* cand_raw;       // [F][max_sel] raw-list index of the quad that decoded
    const uint32_t* first_list;  // work list of k_identify_first (frame << 16 | k)
    uint32_t* retry_list;        // work list of k_identify_retry, filled by k_identify_first
    Counters* counters;          // n_first, n_retry
    A3Pyramid pyr;               // useAruco3Detection (k_identify_*<true>): a candidate's bits come from its pyramid level
    float* cand_conf;            // [F][max_sel] detectMarkersWithConfidence (k_identify_*<PYR, true>), decoded candidates only
};

#define IDENT_WARPS 8    // retry kernel: warps per candidate
#define IDENT0_WARPS 4   // first-attempt kernel: candidates per block (one warp each)

__device__ __forceinline__ void identify_write(const IdentifyArgs& a, size_t fo, size_t o, int id, int rot, int used) {
    a.cand_id[o] = id;
    a.cand_raw[o] = a.fs.raw_of_sorted[fo + used];
    const QuadF use = a.fs.quads[fo + used];
    for (int c = 0; c < 4; c++) {  // correctCornerPosition: std::rotate(begin, begin + 4 - rotation, end)
        a.cand_corners[o * 8 + 2 * c] = use.x[(c + 4 - rot) & 3];
        a.cand_corners[o * 8 + 2 * c + 1] = use.y[(c + 4 - rot) & 3];
    }
}

// cv::aruco tries the selected quad first and then, in order, the "close contours" of its group until one decodes
// (SURVEY A.6).  The first attempt decodes for every real marker, so it gets a kernel of its own with ONE WARP per selected
// candidate -- every candidate of the chunk is in flight at once (a block of 8 warps per candidate held 7 idle warps' worth of
// registers and ran the chunk in five waves).  cand_id = -2 marks the candidates whose first attempt failed and that have
// close contours left to try.
// PYR (useAruco3Detection, aruco3.cuh): the quads are in segmentation-plane coordinates; every attempt for a selected candidate,
// its close contours included, reads the pyramid level its own contour length picks, with the quad scaled to that level.
// CONF (detectMarkersWithConfidence): each decoded candidate's confidence goes to cand_conf, from the cell counts the attempt
// that decoded left in its warp's `hist` (identify.cuh, marker_confidence).
// INV (detectInvertedMarker): every attempt tries both polarities (identify_candidate<CONF, true>); under CONF the counts left in
// `hist` are the chosen polarity's.
template <bool PYR, bool CONF, bool INV>
__device__ __forceinline__ IdentifyResult identify_attempt(const IdentifyArgs& a, const WarpLanes& L, int f, int level, const QuadF& quad, const unsigned long long* dict,
                                                           uint8_t* img, int* hist) {
    if constexpr (PYR) {
        const float s = a3_level_scale(a.pyr.g, level);
        QuadF q;
        for (int c = 0; c < 4; c++) {
            q.x[c] = quad.x[c] * s;
            q.y[c] = quad.y[c] * s;
        }
        return identify_candidate<CONF, INV>(L, a.pyr.plane(f, level), a.pyr.g.lv[level].W, a.pyr.g.lv[level].H, q, a.P, dict, img, hist);
    } else {
        const FrameImg gray{a.src + (size_t)f * a.frame_stride, a.row_stride, a.enc};
        return identify_candidate<CONF, INV>(L, gray, a.W, a.H, quad, a.P, dict, img, hist);
    }
}
template <bool PYR>
__device__ __forceinline__ int identify_level(const IdentifyArgs& a, size_t fo, int si) {
    if constexpr (PYR)
        return a3_level_for(a.pyr.g, a.pyr.raw[fo + a.fs.raw_of_sorted[fo + si]].n_contour);
    else
        return 0;
}

template <bool PYR, bool CONF = false, bool INV = false>
__global__ void __launch_bounds__(IDENT0_WARPS * 32) k_identify_first(const IdentifyArgs a) {
    extern __shared__ unsigned long long sm_dict[];  // n_markers*4 words, then per-warp scratch
    const unsigned int n_first = a.counters->n_first;
    if (blockIdx.x * IDENT0_WARPS >= n_first) return;  // fixed grid, work list: no empty blocks worth mentioning
    const int n_words = a.P.n_markers * 4;
    for (int i = threadIdx.x; i < n_words; i += blockDim.x) sm_dict[i] = __ldg(a.dict + i);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int* hist = reinterpret_cast<int*>(sm_dict + n_words) + warp * 256;
    uint8_t* img = reinterpret_cast<uint8_t*>(reinterpret_cast<int*>(sm_dict + n_words) + IDENT0_WARPS * 256) + warp * (FID_MAX_WARP_SIDE_SQ);
    __syncthreads();
    WarpLanes L;
    for (unsigned int i = blockIdx.x * IDENT0_WARPS + warp; i < n_first; i += gridDim.x * IDENT0_WARPS) {
        const uint32_t rec = a.first_list[i];
        const int f = (int)(rec >> 16), k = (int)(rec & 0xFFFFu);
        const size_t fo = (size_t)f * a.max_raw, o = (size_t)f * a.max_sel + k;
        const int si = a.fs.sel_idx[fo + k];
        const IdentifyResult r = identify_attempt<PYR, CONF, INV>(a, L, f, identify_level<PYR>(a, fo, si), a.fs.quads[fo + si], sm_dict, img, hist);
        __syncwarp();
        if (lane == 0) {
            if (r.id >= 0) {
                identify_write(a, fo, o, r.id, r.rotation, si);
                if constexpr (CONF) a.cand_conf[o] = marker_confidence(hist, a.P, sm_dict[r.id * 4 + r.rotation]);
            } else if (a.fs.close_count[fo + si] > 0) {
                a.cand_id[o] = -2;
                a.retry_list[atomicAdd(&a.counters->n_retry, 1u)] = rec;
            } else {
                a.cand_id[o] = -1;
            }
        }
        if constexpr (CONF) __syncwarp();  // lane 0 is done with the counts before the next candidate overwrites them
    }
}

// One block per candidate whose first attempt failed.  A non-marker group of a dozen nested outlines used to cost a dozen
// identifications back to back in one warp -- the longest chain of the launch.  Here warp w tries attempts 1 + w, 1 + w + 8, ...
// concurrently; the lowest successful attempt wins, which is exactly the sequential first-success rule.
template <bool PYR, bool CONF = false, bool INV = false>
__global__ void __launch_bounds__(IDENT_WARPS * 32) k_identify_retry(const IdentifyArgs a) {
    extern __shared__ unsigned long long sm_dict[];  // n_markers*4 words, then per-warp scratch
    __shared__ int s_best;                            // lowest successful attempt so far
    __shared__ int s_id[IDENT_WARPS], s_rot[IDENT_WARPS], s_att[IDENT_WARPS];
    const unsigned int n_retry = a.counters->n_retry;
    if (blockIdx.x >= n_retry) return;
    const int n_words = a.P.n_markers * 4;
    for (int i = threadIdx.x; i < n_words; i += blockDim.x) sm_dict[i] = __ldg(a.dict + i);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int* hist = reinterpret_cast<int*>(sm_dict + n_words) + warp * 256;
    uint8_t* img = reinterpret_cast<uint8_t*>(reinterpret_cast<int*>(sm_dict + n_words) + IDENT_WARPS * 256) + warp * (FID_MAX_WARP_SIDE_SQ);
    WarpLanes L;
    for (unsigned int i = blockIdx.x; i < n_retry; i += gridDim.x) {
        const uint32_t rec = a.retry_list[i];
        const int f = (int)(rec >> 16), k = (int)(rec & 0xFFFFu);
        const size_t fo = (size_t)f * a.max_raw, o = (size_t)f * a.max_sel + k;
        __syncthreads();  // the previous candidate's result has been read
        if (threadIdx.x == 0) s_best = 0x7fffffff;
        if (lane == 0) s_att[warp] = 0x7fffffff;
        __syncthreads();
        const int si = a.fs.sel_idx[fo + k];
        const int level = identify_level<PYR>(a, fo, si);
        const int nc = a.fs.close_count[fo + si], co = a.fs.close_off[fo + si];
        for (int t = 1 + warp; t <= nc; t += IDENT_WARPS) {
            if (t > *reinterpret_cast<volatile int*>(&s_best)) break;  // an earlier attempt already decoded
            const QuadF quad = a.fs.quads[fo + a.fs.close_idx[fo + co + t - 1]];
            const IdentifyResult r = identify_attempt<PYR, CONF, INV>(a, L, f, level, quad, sm_dict, img, hist);
            __syncwarp();
            if (r.id >= 0) {
                if (lane == 0) {
                    s_id[warp] = r.id;
                    s_rot[warp] = r.rotation;
                    s_att[warp] = t;
                    atomicMin(&s_best, t);
                }
                break;  // later attempts of this warp cannot win
            }
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            int id = -1, rot = 0, att = 0, win_w = 0;
            for (int w = 0; w < IDENT_WARPS; w++)
                if (s_att[w] == s_best && s_best != 0x7fffffff) {
                    id = s_id[w];
                    rot = s_rot[w];
                    att = s_att[w];
                    if constexpr (CONF) win_w = w;
                }
            if (id >= 0) {
                identify_write(a, fo, o, id, rot, a.fs.close_idx[fo + co + att - 1]);
                // the winning warp stopped after its decoding attempt: its hist still holds that attempt's counts
                if constexpr (CONF) a.cand_conf[o] = marker_confidence(reinterpret_cast<int*>(sm_dict + n_words) + win_w * 256, a.P, sm_dict[id * 4 + rot]);
            } else
                a.cand_id[o] = -1;
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// CORNER_REFINE_CONTOUR (contour_refine.cuh), launched only when the method is selected: one CTA per decoded candidate strides
// over the candidate's contour.  Pass 1 finds the positions that coincide with a corner, pass 2 adds every point to the sums
// of the corner seen last before it; the corners are rewritten in place.
struct ContourRefineArgs {
    const int* n_sel;      // [F]
    const int* cand_id;    // [F][max_sel]
    const int* cand_raw;   // [F][max_sel] raw-list index of the quad that decoded
    float* cand_corners;   // [F][max_sel][8], rewritten
    const RawQuad* raw;    // [F][max_raw]: pts_off, n_contour
    const Pt16* points;    // batch point buffer
    int max_raw, max_sel;
};

#define CREFINE_THREADS 128

__global__ void __launch_bounds__(CREFINE_THREADS) k_contour_refine(const ContourRefineArgs a) {
    __shared__ int s_nmatch, s_cidx[4];
    __shared__ int s_mpos[32], s_mcor[32];
    __shared__ long long s_sum[4][6];
    __shared__ int s_ext[4][4];
    const int f = blockIdx.y, k = blockIdx.x, tid = threadIdx.x;
    if (k >= a.n_sel[f]) return;
    const size_t co = (size_t)f * a.max_sel + k;
    if (a.cand_id[co] < 0) return;
    const RawQuad rq = a.raw[(size_t)f * a.max_raw + a.cand_raw[co]];
    const Pt16* pts = a.points + rq.pts_off;
    const int np = rq.n_contour;
    float cx[4], cy[4];
    for (int c = 0; c < 4; c++) {
        cx[c] = a.cand_corners[co * 8 + 2 * c];
        cy[c] = a.cand_corners[co * 8 + 2 * c + 1];
    }
    if (tid == 0) s_nmatch = 0;
    if (tid < 4) s_cidx[tid] = -1;
    if (tid < 24) s_sum[tid / 6][tid % 6] = 0;
    if (tid < 16) s_ext[tid >> 2][tid & 3] = (tid & 1) ? -0x7fffffff : 0x7fffffff;  // min x, max x, min y, max y
    __syncthreads();
    for (int i = tid; i < np; i += CREFINE_THREADS) {
        const float px = (float)pts[i].x, py = (float)pts[i].y;
        for (int j = 0; j < 4; j++)
            if (px == cx[j] && py == cy[j]) {
                const int slot = atomicAdd(&s_nmatch, 1);
                if (slot < 32) {
                    s_mpos[slot] = i;
                    s_mcor[slot] = j;
                }
                atomicMax(&s_cidx[j], i);
            }
    }
    __syncthreads();
    const int nm = s_nmatch;
    if (s_cidx[0] < 0 || s_cidx[1] < 0 || s_cidx[2] < 0 || s_cidx[3] < 0) return;  // cannot happen for a quad of this contour (OpenCV asserts)
    if (nm > 32) {  // a contour that revisits its corners many times: serial
        if (tid == 0) {
            refine_candidate_lines_serial(pts, np, cx, cy);
            for (int c = 0; c < 4; c++) {
                a.cand_corners[co * 8 + 2 * c] = cx[c];
                a.cand_corners[co * 8 + 2 * c + 1] = cy[c];
            }
        }
        return;
    }
    if (tid == 0) {  // order the matches by contour position
        for (int i = 1; i < nm; i++) {
            const int p = s_mpos[i], c = s_mcor[i];
            int j = i - 1;
            for (; j >= 0 && s_mpos[j] > p; j--) {
                s_mpos[j + 1] = s_mpos[j];
                s_mcor[j + 1] = s_mcor[j];
            }
            s_mpos[j + 1] = p;
            s_mcor[j + 1] = c;
        }
    }
    __syncthreads();
    for (int i = tid; i < np; i += CREFINE_THREADS) {
        int g = s_mcor[nm - 1];  // before the first corner: the corner seen last
        for (int q = 0; q < nm && s_mpos[q] <= i; q++) g = s_mcor[q];
        const int x = pts[i].x, y = pts[i].y;
        atomicAdd(reinterpret_cast<unsigned long long*>(&s_sum[g][0]), 1ull);
        atomicAdd(reinterpret_cast<unsigned long long*>(&s_sum[g][1]), (unsigned long long)(long long)x);
        atomicAdd(reinterpret_cast<unsigned long long*>(&s_sum[g][2]), (unsigned long long)(long long)y);
        atomicAdd(reinterpret_cast<unsigned long long*>(&s_sum[g][3]), (unsigned long long)((long long)x * x));
        atomicAdd(reinterpret_cast<unsigned long long*>(&s_sum[g][4]), (unsigned long long)((long long)y * y));
        atomicAdd(reinterpret_cast<unsigned long long*>(&s_sum[g][5]), (unsigned long long)((long long)x * y));
        atomicMin(&s_ext[g][0], x);
        atomicMax(&s_ext[g][1], x);
        atomicMin(&s_ext[g][2], y);
        atomicMax(&s_ext[g][3], y);
    }
    __syncthreads();
    if (tid == 0) {
        LineSums sums[4];
        int cidx[4];
        for (int g = 0; g < 4; g++) {
            sums[g].n = s_sum[g][0];
            sums[g].sx = s_sum[g][1];
            sums[g].sy = s_sum[g][2];
            sums[g].sxx = s_sum[g][3];
            sums[g].syy = s_sum[g][4];
            sums[g].sxy = s_sum[g][5];
            sums[g].minx = s_ext[g][0];
            sums[g].maxx = s_ext[g][1];
            sums[g].miny = s_ext[g][2];
            sums[g].maxy = s_ext[g][3];
            cidx[g] = s_cidx[g];
        }
        corners_from_lines(sums, cidx, cx, cy);
        for (int c = 0; c < 4; c++) {
            a.cand_corners[co * 8 + 2 * c] = cx[c];
            a.cand_corners[co * 8 + 2 * c + 1] = cy[c];
        }
    }
}

// ---------------------------------------------------------------------------------------------------
struct FinishArgs {
    const uint8_t* src;
    size_t row_stride, frame_stride;
    int enc, W, H;
    const int* n_sel;
    const int* cand_id;
    const float* cand_corners;
    FrameScratch fs;  // selected candidates' quads (candidate hierarchy)
    int max_raw;
    int max_sel, max_markers;
    DevParams P;
    const float* subpix_masks;  // windows 1..5 concatenated: offsets 0, 9, 34, 83, 164
    int do_pose;
    Camera cam;
    double fiducial_len;
    int n_override;
    const int32_t* override_ids;
    const double* override_lens;
    int32_t* out_count;     // [F]
    int32_t* out_ids;       // [F][max_markers]
    float* out_corners;     // [F][max_markers][8]
    fid_transform* out_tf;  // [F][max_markers]
    Counters* counters;
};

#define FINISH_THREADS 128
#define FID_MAX_SEL 512  // selected candidates per frame (fid_detector::max_sel)

__device__ __forceinline__ int subpix_mask_offset(int win) {
    int off = 0;
    for (int w = 1; w < win; w++) off += (2 * w + 1) * (2 * w + 1);
    return off;
}

__global__ void __launch_bounds__(FINISH_THREADS) k_finish(const FinishArgs a) {
    __shared__ int s_n;
    __shared__ int s_src[FID_MAX_MARKERS];
    __shared__ short s_parent[FID_MAX_SEL], s_depth[FID_MAX_SEL];
    __shared__ unsigned char s_was[FID_MAX_SEL];
    const int f = blockIdx.x, tid = threadIdx.x;
    const int ns = a.n_sel[f] < FID_MAX_SEL ? a.n_sel[f] : FID_MAX_SEL;
    // OpenCV 4.13 candidate hierarchy (SURVEY A.5): candidates are in descending-perimeter order; the parent of i is the
    // nearest larger candidate whose quad contains all four corners of i.  TWIN: candidate_tree.cuh (tree_parent, tree_levels)
    // states the same loop for k_rejected and the CPU harness; a change here must be made there too, or a candidate ends up both
    // a marker and rejected (tests/test_gpu_batch_refine.py checks markers + rejected == selected on every frame it covers).  It
    // stays inline here because, called through those functions, k_finish compiled to another instruction schedule.
    {
        const size_t fo = (size_t)f * a.max_raw;
        for (int i = tid; i < ns; i += FINISH_THREADS) {
            const QuadF qi = a.fs.quads[fo + a.fs.sel_idx[fo + i]];
            int parent = -1;
            for (int j = i - 1; j >= 0; j--)
                if (quad_inside_quad(qi, a.fs.quads[fo + a.fs.sel_idx[fo + j]])) {
                    parent = j;
                    break;
                }
            s_parent[i] = (short)parent;
            s_depth[i] = 0;
            s_was[i] = 0;
        }
    }
    __syncthreads();
    if (tid == 0) {
        // depth: leaves 0, a parent one more than its deepest child (children have larger indices)
        int max_depth = 0;
        for (int i = ns - 1; i >= 0; i--) {
            const int p = s_parent[i];
            if (p >= 0 && s_depth[p] < s_depth[i] + 1) s_depth[p] = (short)(s_depth[i] + 1);
            max_depth = s_depth[i] > max_depth ? s_depth[i] : max_depth;
        }
        // identification runs level by level, innermost first, `while (counter < ncandidates)`: an identified candidate
        // counts all its not yet visited ancestors, every candidate of a level counts itself once more -- so the loop can end
        // before the outer levels are reached (a marker that encloses an identified marker is then never looked at), but a
        // level that is reached is identified completely.  s_was[i] bit 1 = level reached ("processed").
        int counter = 0;
        for (int depth = 0; depth <= max_depth && counter < ns; depth++) {
            for (int v = 0; v < ns; v++)
                if (s_depth[v] == depth) s_was[v] |= 3;
            for (int v = 0; v < ns; v++) {
                if (s_depth[v] != depth) continue;
                if (a.cand_id[(size_t)f * a.max_sel + v] >= 0)
                    for (int p = s_parent[v]; p != -1; p = s_parent[p])
                        if (!(s_was[p] & 1)) {
                            s_was[p] |= 1;
                            counter++;
                        }
                counter++;
            }
        }
        int n = 0;
        for (int k = 0; k < ns; k++) {
            if (a.cand_id[(size_t)f * a.max_sel + k] < 0 || !(s_was[k] & 2)) continue;
            if (n < a.max_markers && n < FID_MAX_MARKERS) {
                s_src[n++] = k;
            } else {
                atomicOr(&a.counters->overflow, 32u);
            }
        }
        s_n = n;
        a.out_count[f] = n;
    }
    __syncthreads();
    const int n = s_n;
    const FrameImg gray{a.src + (size_t)f * a.frame_stride, a.row_stride, a.enc};
    float* oc = a.out_corners + (size_t)f * a.max_markers * 8;
    // corners (+ sub-pixel refinement), one thread per corner
    for (int c = tid; c < 4 * n; c += FINISH_THREADS) {
        const int m = c >> 2, ci = c & 3;
        const size_t src = ((size_t)f * a.max_sel + s_src[m]) * 8;
        float x = a.cand_corners[src + 2 * ci], y = a.cand_corners[src + 2 * ci + 1];
        if (a.P.corner_refine == 1) {
            QuadF q;
            for (int k = 0; k < 4; k++) {
                q.x[k] = a.cand_corners[src + 2 * k];
                q.y[k] = a.cand_corners[src + 2 * k + 1];
            }
            const float module = quad_module_size(q, a.P.marker_size, a.P.marker_border_bits);
            int win = __float2int_rn((float)a.P.rel_refine_win * module);
            win = win < 1 ? 1 : win;
            win = win < a.P.refine_win ? win : a.P.refine_win;
            float patch[(2 * FID_SUBPIX_MAX_WIN + 3) * (2 * FID_SUBPIX_MAX_WIN + 3)];
            corner_subpix(gray, a.W, a.H, &x, &y, win, a.subpix_masks + subpix_mask_offset(win), a.P.refine_max_iter,
                          a.P.refine_min_acc * a.P.refine_min_acc, patch);
        }
        oc[(size_t)m * 8 + 2 * ci] = x;
        oc[(size_t)m * 8 + 2 * ci + 1] = y;
    }
    for (int m = tid; m < n; m += FINISH_THREADS) a.out_ids[(size_t)f * a.max_markers + m] = a.cand_id[(size_t)f * a.max_sel + s_src[m]];
    __syncthreads();
    // pose, one thread per marker
    if (a.do_pose) {
        for (int m = tid; m < n; m += FINISH_THREADS) {
            const int id = a.cand_id[(size_t)f * a.max_sel + s_src[m]];
            double len = (double)(float)a.fiducial_len;  // estimatePoseSingleMarkers((float)fiducial_len, ...)  :425
            for (int k = 0; k < a.n_override; k++)
                if (a.override_ids[k] == id) len = a.override_lens[k];
            PoseOut po;
            solve_marker_pose(oc + (size_t)m * 8, a.cam, (float)len, a.fiducial_len, &po);
            fid_transform t;
            t.fiducial_id = id;
            t.reserved = po.lm_iters;
            for (int k = 0; k < 3; k++) {
                t.translation[k] = po.tvec[k];
                t.rvec[k] = po.rvec[k];
            }
            for (int k = 0; k < 4; k++) t.rotation[k] = po.quat[k];
            t.image_error = po.image_error;
            t.object_error = po.object_error;
            t.fiducial_area = po.area;
            a.out_tf[(size_t)f * a.max_markers + m] = t;
        }
    }
}

// detectMarkers' rejectedImgPoints (DESIGN.md finding 11): the selected candidates that are not markers -- not decoded, or decoded
// on a level of the candidate hierarchy that identification never reached -- in selection order (descending perimeter), each with
// the selected quad's own corners (integers, clockwise, neither rotated nor refined).  One block per frame, after k_finish.
// detectMarkersWithConfidence (fid_set_marker_confidence / fid_detect_with_confidence): the confidences k_identify_*<PYR, true>
// wrote per candidate, in k_finish's marker order -- the decoded candidates on a level identification reached, in selection order,
// at most max_markers.  The hierarchy is restated through candidate_tree.cuh as k_rejected does, so that k_finish stays as it is.
// One block per frame, after k_finish.
struct ConfGatherArgs {
    const int* n_sel;
    const int* cand_id;
    const float* cand_conf;  // [F][max_sel]
    FrameScratch fs;
    int max_raw, max_sel, max_markers;
    float* out_conf;         // [F][max_markers]
};

__global__ void __launch_bounds__(FINISH_THREADS) k_conf_gather(const ConfGatherArgs a) {
    __shared__ short s_parent[FID_MAX_SEL], s_depth[FID_MAX_SEL];
    __shared__ unsigned char s_was[FID_MAX_SEL];
    const int f = blockIdx.x, tid = threadIdx.x;
    const int ns = a.n_sel[f] < FID_MAX_SEL ? a.n_sel[f] : FID_MAX_SEL;
    const size_t fo = (size_t)f * a.max_raw;
    const int* cand_id = a.cand_id + (size_t)f * a.max_sel;
    for (int i = tid; i < ns; i += FINISH_THREADS) {
        s_parent[i] = (short)tree_parent(a.fs.quads[fo + a.fs.sel_idx[fo + i]], i, [&](int j) { return a.fs.quads[fo + a.fs.sel_idx[fo + j]]; });
        s_depth[i] = 0;
        s_was[i] = 0;
    }
    __syncthreads();
    if (tid == 0) {
        tree_levels(ns, s_parent, s_depth, s_was, [&](int v) { return cand_id[v] >= 0; });
        const int cap = a.max_markers < FID_MAX_MARKERS ? a.max_markers : FID_MAX_MARKERS;
        int n = 0;
        for (int k = 0; k < ns && n < cap; k++)
            if (cand_id[k] >= 0 && (s_was[k] & 2)) a.out_conf[(size_t)f * a.max_markers + n++] = a.cand_conf[(size_t)f * a.max_sel + k];
    }
}

struct RejectedArgs {
    const int* n_sel;
    const int* cand_id;
    FrameScratch fs;
    int max_raw, max_sel;
    int32_t* n_rej;  // [F]
    float* rej;      // [F][max_sel][8]
};

__global__ void __launch_bounds__(FINISH_THREADS) k_rejected(const RejectedArgs a) {
    __shared__ short s_parent[FID_MAX_SEL], s_depth[FID_MAX_SEL];
    __shared__ unsigned char s_was[FID_MAX_SEL];
    __shared__ short s_src[FID_MAX_SEL];
    __shared__ int s_n;
    const int f = blockIdx.x, tid = threadIdx.x;
    const int ns = a.n_sel[f] < FID_MAX_SEL ? a.n_sel[f] : FID_MAX_SEL;
    const size_t fo = (size_t)f * a.max_raw;
    const int* cand_id = a.cand_id + (size_t)f * a.max_sel;
    for (int i = tid; i < ns; i += FINISH_THREADS) {
        s_parent[i] = (short)tree_parent(a.fs.quads[fo + a.fs.sel_idx[fo + i]], i, [&](int j) { return a.fs.quads[fo + a.fs.sel_idx[fo + j]]; });
        s_depth[i] = 0;
        s_was[i] = 0;
    }
    __syncthreads();
    if (tid == 0) {
        tree_levels(ns, s_parent, s_depth, s_was, [&](int v) { return cand_id[v] >= 0; });
        int n = 0;
        for (int k = 0; k < ns; k++)
            if (cand_id[k] < 0 || !(s_was[k] & 2)) s_src[n++] = (short)k;
        s_n = n;
        a.n_rej[f] = n;
    }
    __syncthreads();
    float* out = a.rej + (size_t)f * a.max_sel * 8;
    for (int c = tid; c < 4 * s_n; c += FINISH_THREADS) {
        const QuadF q = a.fs.quads[fo + a.fs.sel_idx[fo + s_src[c >> 2]]];
        out[2 * c] = q.x[c & 3];
        out[2 * c + 1] = q.y[c & 3];
    }
}

// Poses of the markers k_marker_refine appended in a batch: slots [count[f] - n_rec[f], count[f]) of each frame, solved as k_finish
// solves the detected ones.  One block per frame, one thread per marker.
struct RecoveredPoseArgs {
    const int32_t* count;  // [F] after refinement
    const int32_t* n_rec;  // [F]
    const int32_t* ids;
    const float* corners;
    int max_markers;
    Camera cam;
    double fiducial_len;
    int n_override;
    const int32_t* override_ids;
    const double* override_lens;
    fid_transform* out_tf;
};

__global__ void __launch_bounds__(32) k_recovered_pose(const RecoveredPoseArgs a) {
    const int f = blockIdx.x;
    const int n = a.count[f];
    for (int m = n - a.n_rec[f] + (int)threadIdx.x; m < n; m += 32) {
        const size_t o = (size_t)f * a.max_markers + m;
        const int id = a.ids[o];
        double len = (double)(float)a.fiducial_len;
        for (int k = 0; k < a.n_override; k++)
            if (a.override_ids[k] == id) len = a.override_lens[k];
        PoseOut po;
        solve_marker_pose(a.corners + o * 8, a.cam, (float)len, a.fiducial_len, &po);
        fid_transform t;
        t.fiducial_id = id;
        t.reserved = po.lm_iters;
        for (int k = 0; k < 3; k++) {
            t.translation[k] = po.tvec[k];
            t.rvec[k] = po.rvec[k];
        }
        for (int k = 0; k < 4; k++) t.rotation[k] = po.quat[k];
        t.image_error = po.image_error;
        t.object_error = po.object_error;
        t.fiducial_area = po.area;
        a.out_tf[o] = t;
    }
}

// Pose only (fid_pose): one thread per marker of a single list.
struct PoseArgs {
    int n;
    const int32_t* ids;
    const float* corners;
    Camera cam;
    double fiducial_len;
    int n_override;
    const int32_t* override_ids;
    const double* override_lens;
    fid_transform* out;
};

__global__ void __launch_bounds__(64) k_pose(const PoseArgs a) {
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= a.n) return;
    const int id = a.ids[m];
    double len = (double)(float)a.fiducial_len;
    for (int k = 0; k < a.n_override; k++)
        if (a.override_ids[k] == id) len = a.override_lens[k];
    PoseOut po;
    solve_marker_pose(a.corners + (size_t)m * 8, a.cam, (float)len, a.fiducial_len, &po);
    fid_transform t;
    t.fiducial_id = id;
    t.reserved = po.lm_iters;
    for (int k = 0; k < 3; k++) {
        t.translation[k] = po.tvec[k];
        t.rvec[k] = po.rvec[k];
    }
    for (int k = 0; k < 4; k++) t.rotation[k] = po.quat[k];
    t.image_error = po.image_error;
    t.object_error = po.object_error;
    t.fiducial_area = po.area;
    a.out[m] = t;
}


// ---------------------------------------------------------------------------------------------------
// Both planar pose hypotheses (ippe.cuh), an opt-in stage of its own so that k_finish and the default pipeline stay as they are.
__device__ __forceinline__ void pack_hypotheses(int id, const PoseHypOut& ho, struct fid_pose_hypotheses* r) {
    struct fid_pose_hypotheses t;
    t.fiducial_id = id;
    t.n = ho.n;
    t.iterative_match = ho.iterative_match;
    t.reserved = 0;
    for (int s = 0; s < 2; s++) {
        for (int k = 0; k < 3; k++) {
            t.rvec[s][k] = ho.rvec[s][k];
            t.tvec[s][k] = ho.tvec[s][k];
        }
        t.rms[s] = ho.rms[s];
    }
    *r = t;
}

__device__ __forceinline__ double marker_len_of(int id, double fiducial_len, int n_override, const int32_t* override_ids, const double* override_lens) {
    double len = (double)(float)fiducial_len;  // as k_finish / k_pose
    for (int k = 0; k < n_override; k++)
        if (override_ids[k] == id) len = override_lens[k];
    return len;
}

struct PoseHypArgs {
    int nf, max_markers;
    const int32_t* count;         // [F]                   k_finish's outputs
    const float* corners;         // [F][max_markers][8]
    const fid_transform* tf;      // [F][max_markers]      the ITERATIVE pose (rvec) and the id
    Camera cam;
    double fiducial_len;
    int n_override;
    const int32_t* override_ids;
    const double* override_lens;
    struct fid_pose_hypotheses* out;  // [F][max_markers]; slots past count[f] are not written
};

#define POSE_HYP_THREADS 32

// One block per frame, one thread per marker.
__global__ void __launch_bounds__(POSE_HYP_THREADS) k_pose_hypotheses(const PoseHypArgs a) {
    const int f = blockIdx.x;
    const int n = a.count[f];
    for (int m = threadIdx.x; m < n; m += POSE_HYP_THREADS) {
        const size_t o = (size_t)f * a.max_markers + m;
        const fid_transform& t = a.tf[o];
        const int id = t.fiducial_id;
        const double rit[3] = {t.rvec[0], t.rvec[1], t.rvec[2]};
        PoseHypOut ho;
        solve_marker_hypotheses(a.corners + o * 8, a.cam, (float)marker_len_of(id, a.fiducial_len, a.n_override, a.override_ids, a.override_lens), rit, &ho);
        pack_hypotheses(id, ho, a.out + o);
    }
}

// Host corners (fid_pose_hypotheses): one thread per marker of a single list; the ITERATIVE pose is solved here as k_pose does.
struct PoseHypListArgs {
    int n;
    const int32_t* ids;
    const float* corners;
    Camera cam;
    double fiducial_len;
    int n_override;
    const int32_t* override_ids;
    const double* override_lens;
    struct fid_pose_hypotheses* out;
};

__global__ void __launch_bounds__(64) k_pose_hypotheses_list(const PoseHypListArgs a) {
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= a.n) return;
    const int id = a.ids[m];
    const float len = (float)marker_len_of(id, a.fiducial_len, a.n_override, a.override_ids, a.override_lens);
    PoseOut po;
    solve_marker_pose(a.corners + (size_t)m * 8, a.cam, len, a.fiducial_len, &po);
    PoseHypOut ho;
    solve_marker_hypotheses(a.corners + (size_t)m * 8, a.cam, len, po.rvec, &ho);
    pack_hypotheses(id, ho, a.out + m);
}

// ---------------------------------------------------------------------------------------------------
// One pose per board (board_pnp.cuh), an opt-in stage of its own so that k_finish and the default pipeline stay as they are.
struct BoardPoseArgs {
    int max_markers, n_boards;
    const int32_t* count;         // [F]                   k_finish's outputs (or one host list)
    const int32_t* ids;           // [F][max_markers]
    const float* corners;         // [F][max_markers][8]
    const int32_t* board_off;     // [n_boards + 1]        board b = rows board_off[b] .. board_off[b + 1] of the three tables
    const int32_t* board_keys;    //                       its ids, sorted
    const int32_t* board_marker;  //                       the marker (row within the board) of each sorted id
    const float* board_obj;       // [rows][4][3]          object points, in the board's own marker order
    const int32_t* run;           // [F][FID_MAX_DICTIONARIES + 1] family runs of the merged list (k_dict_merge), or nullptr: every marker
    int32_t family[FID_MAX_BOARDS];  //                    each board's dictionary index (read with run only)
    Camera cam;
    fid_board_pose* out;          // [F][n_boards]
};

// Multi-dictionary mode: a family's markers are one contiguous run of the frame's merged list (DESIGN.md finding 19), so a stage
// bound to family k reads that run as the frame's list: corners[di == k], ids[di == k] in list order.
__device__ __forceinline__ void family_run(const int32_t* run, int f, int family, const int32_t** ids, const float** corners, int* n) {
    const int32_t* r = run + (size_t)f * (FID_MAX_DICTIONARIES + 1) + family;
    *ids += r[0];
    *corners += (size_t)r[0] * 8;
    *n = r[1] - r[0];
}

#define BOARD_POSE_MAX_POINTS (4 * FID_MAX_MARKERS)

// One warp per (frame, board): lanes binary-search the board's sorted ids for 32 detections at a time, a ballot / popc prefix
// keeps Board::matchImagePoints's order while the matched points are staged in shared memory, then the warp solves the pose.
__global__ void __launch_bounds__(FID_BOARD_LANES) k_board_pose(const BoardPoseArgs a) {
    __shared__ float s_obj[BOARD_POSE_MAX_POINTS * 3];
    __shared__ float s_img[BOARD_POSE_MAX_POINTS * 2];
    __shared__ double s_mn[BOARD_POSE_MAX_POINTS * 2];
    const int f = blockIdx.x / a.n_boards, b = blockIdx.x % a.n_boards;
    const int lane = threadIdx.x;
    int n = min(a.count[f], FID_MAX_MARKERS);
    const int off = a.board_off[b], nb = a.board_off[b + 1] - off;
    const int32_t* ids = a.ids + (size_t)f * a.max_markers;
    const float* corners = a.corners + (size_t)f * a.max_markers * 8;
    if (a.run) family_run(a.run, f, a.family[b], &ids, &corners, &n);
    int m = 0;
    for (int j0 = 0; j0 < n; j0 += FID_BOARD_LANES) {
        const int j = j0 + lane;
        const int k = j < n ? board_find(a.board_keys + off, nb, ids[j]) : -1;
        const unsigned hit = __ballot_sync(0xffffffffu, k >= 0);
        if (k >= 0) {
            const int pos = m + __popc(hit & ((1u << lane) - 1u));
            const float* o = a.board_obj + (size_t)(off + a.board_marker[off + k]) * 12;
            for (int c = 0; c < 12; c++) s_obj[pos * 12 + c] = o[c];
            for (int c = 0; c < 8; c++) s_img[pos * 8 + c] = corners[(size_t)j * 8 + c];
        }
        m += __popc(hit);
    }
    __syncwarp();
    BoardPoseOut po;
    solve_board_pose(4 * m, s_obj, s_img, s_mn, a.cam, &po);
    if (lane == 0) {
        fid_board_pose r;
        r.board = b;
        r.status = po.status;
        r.n_markers = m;
        r.n_points = po.n_points;
        for (int k = 0; k < 3; k++) {
            r.rvec[k] = po.rvec[k];
            r.tvec[k] = po.tvec[k];
        }
        for (int k = 0; k < 4; k++) r.rotation[k] = po.quat[k];
        r.image_error = po.image_error;
        a.out[(size_t)f * a.n_boards + b] = r;
    }
}

// ---------------------------------------------------------------------------------------------------
// ChArUco corners and pose (charuco.cuh), an opt-in stage of its own after every other stage.
struct CharucoBoardDev {
    int n_markers, n_corners;
    int marker_off, corner_off;  // rows of the marker tables / of the corner tables; corner_off is also the board's first output slot
    int min_markers, check_markers;
    int family;                  // its dictionary index (read with CharucoArgs::run only)
};

struct CharucoArgs {
    const uint8_t* src;
    size_t row_stride, frame_stride;
    int enc, W, H;
    int max_markers;
    const int32_t* count;    // [F]                     k_finish's outputs (or one host list)
    const int32_t* ids;      // [F][max_markers]
    const float* corners;    // [F][max_markers][8]
    int n_boards, n_slots;
    const CharucoBoardDev* boards;
    const int32_t *keys, *marker_of, *board_ids;  // marker tables, see CharucoView
    const float* obj;
    const float* chess;                           // corner tables
    const int32_t *near_n, *near_idx, *near_corner;
    const float* masks;      // charuco_subpix_masks
    const int32_t* run;      // as BoardPoseArgs; each board's family is CharucoBoardDev::family
    int win_default, max_iters;
    double eps_sq;
    int has_cam;
    Camera cam;
    fid_charuco_result* out;  // [F][n_boards]
    int32_t* out_ids;         // [F][n_slots]
    float* out_xy;            // [F][n_slots][2]
};

#define CHARUCO_THREADS 128
#define CHARUCO_PTS (4 * FID_MAX_MARKERS > FID_MAX_CHARUCO_CORNERS ? 4 * FID_MAX_MARKERS : FID_MAX_CHARUCO_CORNERS)
// dynamic shared memory: points of the two solvePnP calls (obj, img, normalised), detection ids and board markers, corner positions,
// their output slots and the ids in output order
#define CHARUCO_SMEM (CHARUCO_PTS * (3 * 4 + 2 * 4 + 2 * 8) + FID_MAX_MARKERS * 2 * 4 + FID_MAX_CHARUCO_CORNERS * (2 * 4 + 4 + 4))

__device__ __forceinline__ void charuco_pack(const BoardPoseOut& po, int status, fid_charuco_result* r) {
    r->status = status;
    for (int k = 0; k < 3; k++) {
        r->rvec[k] = status == 1 ? po.rvec[k] : 0.0;
        r->tvec[k] = status == 1 ? po.tvec[k] : 0.0;
    }
    for (int k = 0; k < 4; k++) r->rotation[k] = status == 1 ? po.quat[k] : 0.0;
    r->image_error = status == 1 ? po.image_error : 0.0;
}

// One block per (frame, board).  Warp 0 solves the approximate pose over the board's markers (with a camera), threads then take one
// chessboard corner at a time (position, window, border and minMarkers filters, cornerSubPix), the block runs checkBoard, the
// corners are compacted in ascending id, and warp 0 solves the board pose.
__global__ void __launch_bounds__(CHARUCO_THREADS) k_charuco(const CharucoArgs a) {
    extern __shared__ __align__(16) unsigned char charuco_smem[];
    double* s_mn = (double*)charuco_smem;
    float* s_obj = (float*)(s_mn + 2 * CHARUCO_PTS);
    float* s_img = s_obj + 3 * CHARUCO_PTS;
    int32_t* s_ids = (int32_t*)(s_img + 2 * CHARUCO_PTS);
    int32_t* s_k = s_ids + FID_MAX_MARKERS;
    float* s_xy = (float*)(s_k + FID_MAX_MARKERS);
    int32_t* s_slot = (int32_t*)(s_xy + 2 * FID_MAX_CHARUCO_CORNERS);
    int32_t* s_cid = s_slot + FID_MAX_CHARUCO_CORNERS;
    __shared__ double s_p[6];
    __shared__ int s_m, s_n;
    const int f = blockIdx.x / a.n_boards, b = blockIdx.x % a.n_boards;
    const int tid = threadIdx.x, lane = tid & 31;
    const CharucoBoardDev bd = a.boards[b];
    const CharucoView B{bd.n_markers, bd.n_corners, bd.min_markers, bd.check_markers, a.keys + bd.marker_off, a.marker_of + bd.marker_off, a.board_ids + bd.marker_off,
                        a.obj + (size_t)bd.marker_off * 12, a.chess + (size_t)bd.corner_off * 3, a.near_n + bd.corner_off, a.near_idx + 2 * bd.corner_off,
                        a.near_corner + 2 * bd.corner_off};
    int n = min(a.count[f], FID_MAX_MARKERS);
    const int32_t* ids = a.ids + (size_t)f * a.max_markers;
    const float* corners = a.corners + (size_t)f * a.max_markers * 8;
    if (a.run) family_run(a.run, f, bd.family, &ids, &corners, &n);
    for (int j = tid; j < n; j += CHARUCO_THREADS) {
        s_ids[j] = ids[j];
        const int k = board_find(B.keys, B.n_markers, ids[j]);
        s_k[j] = k < 0 ? -1 : B.marker_of[k];
    }
    __syncthreads();
    // 1. approximate pose (matchImagePoints over the markers in detection order, solvePnP)
    if (a.has_cam && tid < 32) {
        int m = 0;
        for (int j0 = 0; j0 < n; j0 += 32) {
            const int j = j0 + lane;
            const int k = j < n ? s_k[j] : -1;
            const unsigned hit = __ballot_sync(0xffffffffu, k >= 0);
            if (k >= 0) {
                const int pos = m + __popc(hit & ((1u << lane) - 1u));
                for (int c = 0; c < 12; c++) s_obj[pos * 12 + c] = B.obj[(size_t)k * 12 + c];
                for (int c = 0; c < 8; c++) s_img[pos * 8 + c] = corners[(size_t)j * 8 + c];
            }
            m += __popc(hit);
        }
        __syncwarp();
        if (m > 0) {
            BoardPoseOut po;
            solve_board_pose(4 * m, s_obj, s_img, s_mn, a.cam, &po);
            if (lane == 0)
                for (int k = 0; k < 3; k++) {
                    s_p[k] = po.rvec[k];
                    s_p[3 + k] = po.tvec[k];
                }
        }
        if (lane == 0) s_m = m;
    }
    __syncthreads();
    const bool any = !a.has_cam || s_m > 0;
    double p[6], R[9];
    if (a.has_cam && any) {
        for (int k = 0; k < 6; k++) p[k] = s_p[k];
        rodrigues_v2m(p, R, nullptr);
    }
    // 2. per corner: position, window, filters, cornerSubPix
    const FrameImg gray{a.src + (size_t)f * a.frame_stride, a.row_stride, a.enc};
    for (int i = tid; i < B.n_corners; i += CHARUCO_THREADS) {
        float xy[2] = {-1.f, -1.f};
        bool keep = false;
        if (any) {
            if (a.has_cam) charuco_project(B, i, R, p, a.cam, xy);
            else charuco_corner_local(B, i, n, s_ids, corners, xy);
            keep = charuco_inside(xy, a.W, a.H) && charuco_marker_count(B, i, n, s_ids) >= B.min_markers;
            if (keep) {
                const int win = charuco_window(B, i, xy, n, s_ids, corners);
                float patch[(2 * FID_CHARUCO_MAX_WIN + 3) * (2 * FID_CHARUCO_MAX_WIN + 3)];
                charuco_refine(gray, a.W, a.H, xy, win < 0 ? a.win_default : win, a.masks, a.max_iters, a.eps_sq, patch);
            }
        }
        s_xy[2 * i] = xy[0];
        s_xy[2 * i + 1] = xy[1];
        s_slot[i] = keep ? 1 : 0;
    }
    __syncthreads();
    // 3. checkBoard over the corners kept
    int bad = 0;
    if (B.check_markers)
        for (int i = tid; i < B.n_corners; i += CHARUCO_THREADS)
            if (s_slot[i] && !charuco_check_corner(B, i, s_xy + 2 * i, n, s_ids, s_k, corners)) bad = 1;
    bad = __syncthreads_or(bad);
    // 4. compaction in ascending id
    if (tid == 0) {
        int q = 0;
        for (int i = 0; i < B.n_corners; i++) {
            const int keep = s_slot[i] && !bad;
            s_slot[i] = keep ? q : -1;
            if (keep) s_cid[q++] = i;
        }
        s_n = q;
    }
    __syncthreads();
    const int nc = s_n;
    int32_t* oid = a.out_ids + (size_t)f * a.n_slots + bd.corner_off;
    float* oxy = a.out_xy + ((size_t)f * a.n_slots + bd.corner_off) * 2;
    for (int q = tid; q < B.n_corners; q += CHARUCO_THREADS) {
        if (q < nc) {
            const int i = s_cid[q];
            oid[q] = i;
            oxy[2 * q] = s_img[2 * q] = s_xy[2 * i];
            oxy[2 * q + 1] = s_img[2 * q + 1] = s_xy[2 * i + 1];
            for (int k = 0; k < 3; k++) s_obj[3 * q + k] = B.chess[3 * i + k];
        } else {
            oid[q] = -1;
            oxy[2 * q] = oxy[2 * q + 1] = -1.f;
        }
    }
    __syncthreads();
    // 5. the board pose
    if (tid < 32) {
        BoardPoseOut po{};
        int status = 0;
        if (bad) status = -3;
        else if (a.has_cam && nc >= 4) {
            if (charuco_collinear(B, nc, s_cid)) status = -2;
            else {
                solve_board_pose(nc, s_obj, s_img, s_mn, a.cam, &po);
                status = po.status;  // 1: the chessboard corners lie in z = 0, so the planar branch runs, which always solves
            }
        }
        if (lane == 0) {
            fid_charuco_result r;
            r.board = b;
            r.n_corners = nc;
            r.corner_offset = bd.corner_off;
            charuco_pack(po, status, &r);
            a.out[(size_t)f * a.n_boards + b] = r;
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// Recovery of missed board markers (marker_refine.cuh): the marker boards, then the ChArUco boards, one refineDetectedMarkers call
// after another, each on the lists the previous one left.
struct MarkerRefineArgs {
    const uint8_t* src;
    size_t row_stride, frame_stride;
    int enc, W, H;
    DevParams P;
    const unsigned long long* dict;  // n_markers x 4 words
    const float* subpix_masks;       // windows 1..5 (k_finish's table)
    MarkerRefineParams rp;
    int n_boards;                    // marker boards, tables as BoardPoseArgs
    const int32_t *board_off, *board_keys, *board_marker;
    const float* board_obj;
    int n_charuco;                   // ChArUco boards, tables as CharucoArgs
    const CharucoBoardDev* ch_boards;
    const int32_t *ch_keys, *ch_marker;
    const float* ch_obj;
    int has_cam;
    Camera cam;
    const int32_t* n_rej;            // [F]
    const float* rej;                // [F][max_rej][8]
    int max_rej, max_markers;
    int32_t* count;                  // [F]                    the detections; recovered markers are appended
    int32_t* ids;                    // [F][max_markers]
    float* corners;                  // [F][max_markers][8]
    int32_t* n_rec;                  // [F]
    int32_t* rec_idx;                // [F][max_markers]       index into the frame's rejected list
    int32_t* rec_board;              // [F][max_markers]       marker board b, or FID_MAX_BOARDS + ChArUco board c
    uint32_t* overflow;              // bit 32: a recovered marker found no slot below max_markers; refinement of the frame stops there
};

#define MREFINE_THREADS 128
#define FID_MAX_BOARD_ROWS 4096
// dynamic shared memory: the matched points of solvePnP (normalised, object, image), board ids in board order, detected-row bits,
// the rejected candidates taken, and one warp's bit-extraction scratch
#define MREFINE_SMEM (4 * FID_MAX_MARKERS * (2 * 8 + 3 * 4 + 2 * 4) + FID_MAX_BOARD_ROWS * 4 + FID_MAX_BOARD_ROWS / 8 + FID_MAX_REJECTED + 256 * 4 + FID_MAX_WARP_SIDE_SQ)

// One block per frame.  Per board: threads find the detected board rows, warp 0 solves the pose (or the homography), then chunks of
// board rows are projected and screened by the threads, compacted in board order, and warp 0 replays the greedy matching over the
// survivors with warp-cooperative bit extraction.
__global__ void __launch_bounds__(MREFINE_THREADS) k_marker_refine(const MarkerRefineArgs a) {
    extern __shared__ __align__(16) unsigned char mrefine_smem[];
    double* s_mn = (double*)mrefine_smem;
    float* s_obj = (float*)(s_mn + 2 * 4 * FID_MAX_MARKERS);
    float* s_img = s_obj + 3 * 4 * FID_MAX_MARKERS;
    int32_t* s_rowid = (int32_t*)(s_img + 2 * 4 * FID_MAX_MARKERS);
    uint32_t* s_found = (uint32_t*)(s_rowid + FID_MAX_BOARD_ROWS);
    int* s_hist = (int*)(s_found + FID_MAX_BOARD_ROWS / 32);
    uint8_t* s_taken = (uint8_t*)(s_hist + 256);
    uint8_t* s_warp = s_taken + FID_MAX_REJECTED;
    __shared__ int32_t s_detrow[FID_MAX_MARKERS], s_first[FID_MAX_MARKERS], s_hrow[FID_MAX_MARKERS], s_hdet[FID_MAX_MARKERS];
    __shared__ int32_t s_surv[MREFINE_THREADS];
    __shared__ float s_proj[MREFINE_THREADS][8];
    __shared__ double s_p[9];
    __shared__ int s_n, s_nrec, s_ntaken, s_ok, s_m, s_ns, s_full, s_wcnt[MREFINE_THREADS / 32];
    const int f = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n_rej = min(a.n_rej[f], min(a.max_rej, FID_MAX_REJECTED));
    const float* rej = a.rej + (size_t)f * a.max_rej * 8;
    int32_t* ids = a.ids + (size_t)f * a.max_markers;
    float* corners = a.corners + (size_t)f * a.max_markers * 8;
    const FrameImg gray{a.src + (size_t)f * a.frame_stride, a.row_stride, a.enc};
    for (int j = tid; j < n_rej; j += MREFINE_THREADS) s_taken[j] = 0;
    if (tid == 0) {
        s_n = min(a.count[f], min(a.max_markers, FID_MAX_MARKERS));
        s_nrec = 0;
        s_ntaken = 0;
        s_full = 0;
    }
    for (int bi = 0; bi < a.n_boards + a.n_charuco; bi++) {
        __syncthreads();
        if (s_full) break;
        const int n0 = s_n;
        if (n0 == 0 || s_ntaken == n_rej) continue;  // refineDetectedMarkers returns at once
        RefineBoardView B;
        int label;
        if (bi < a.n_boards) {
            const int off = a.board_off[bi];
            B = RefineBoardView{a.board_off[bi + 1] - off, a.board_keys + off, a.board_marker + off, a.board_obj + (size_t)off * 12};
            label = bi;
        } else {
            const CharucoBoardDev bd = a.ch_boards[bi - a.n_boards];
            B = RefineBoardView{bd.n_markers, a.ch_keys + bd.marker_off, a.ch_marker + bd.marker_off, a.ch_obj + (size_t)bd.marker_off * 12};
            label = FID_MAX_BOARDS + bi - a.n_boards;
        }
        // 1. board ids in board order, the detected rows (against the detections this call starts with)
        for (int k = tid; k < B.n; k += MREFINE_THREADS) s_rowid[B.marker_of[k]] = B.keys[k];
        for (int w = tid; w < (B.n + 31) / 32; w += MREFINE_THREADS) s_found[w] = 0;
        if (tid == 0) s_m = 0;
        __syncthreads();
        for (int j = tid; j < n0; j += MREFINE_THREADS) {
            const int k = board_find(B.keys, B.n, ids[j]);
            const int row = k < 0 ? -1 : B.marker_of[k];
            s_detrow[j] = row;
            if (row >= 0) atomicOr(&s_found[row >> 5], 1u << (row & 31));
        }
        __syncthreads();
        if (!a.has_cam) {  // the homography's points: the first detection of every detected board row, in board order
            for (int j = tid; j < n0; j += MREFINE_THREADS) {
                const int row = s_detrow[j];
                bool first = row >= 0;
                for (int i = 0; i < j && first; i++) first = s_detrow[i] != row;
                s_first[j] = first;
            }
            __syncthreads();
            for (int j = tid; j < n0; j += MREFINE_THREADS) {
                if (!s_first[j]) continue;
                const int row = s_detrow[j];
                int rank = 0;
                for (int i = 0; i < n0; i++) rank += s_first[i] && s_detrow[i] < row;
                s_hrow[rank] = row;
                s_hdet[rank] = j;
                atomicAdd(&s_m, 1);
            }
            __syncthreads();
        }
        // 2. the prediction: warp 0 solves the board pose or the homography
        if (warp == 0) {
            int ok = 0;
            if (a.has_cam) {
                int m = 0;
                for (int j0 = 0; j0 < n0; j0 += 32) {
                    const int j = j0 + lane;
                    const int row = j < n0 ? s_detrow[j] : -1;
                    const unsigned hit = __ballot_sync(0xffffffffu, row >= 0);
                    if (row >= 0) {
                        const int pos = m + __popc(hit & ((1u << lane) - 1u));
                        for (int c = 0; c < 12; c++) s_obj[pos * 12 + c] = B.obj[(size_t)row * 12 + c];
                        for (int c = 0; c < 8; c++) s_img[pos * 8 + c] = corners[(size_t)j * 8 + c];
                    }
                    m += __popc(hit);
                }
                __syncwarp();
                if (m > 0) {
                    BoardPoseOut po;
                    solve_board_pose(4 * m, s_obj, s_img, s_mn, a.cam, &po);
                    ok = po.status == 1;  // -1: cv2's solvePnP raises
                    if (ok && lane == 0)
                        for (int k = 0; k < 3; k++) {
                            s_p[k] = po.rvec[k];
                            s_p[3 + k] = po.tvec[k];
                        }
                }
            } else {
                bool flat = true;  // cv2 asserts that every board point has the z of the first
                for (int i = lane; i < 4 * B.n; i += 32) flat = flat && B.obj[3 * i + 2] == B.obj[2];
                const int m = s_m;
                if (__all_sync(0xffffffffu, flat) && m > 0) {
                    double Hm[9];
                    ok = board_homography(4 * m, [&](int i, float s[2], float d[2]) {
                        const int row = s_hrow[i >> 2], c = i & 3;
                        s[0] = B.obj[(size_t)row * 12 + 3 * c];
                        s[1] = B.obj[(size_t)row * 12 + 3 * c + 1];
                        d[0] = corners[(size_t)s_hdet[i >> 2] * 8 + 2 * c];
                        d[1] = corners[(size_t)s_hdet[i >> 2] * 8 + 2 * c + 1];
                    }, Hm);
                    if (ok && lane == 0)
                        for (int k = 0; k < 9; k++) s_p[k] = Hm[k];
                }
            }
            if (lane == 0) s_ok = ok;
        }
        __syncthreads();
        if (!s_ok) continue;
        double p[9], R[9];
        for (int k = 0; k < 9; k++) p[k] = s_p[k];
        if (a.has_cam) rodrigues_v2m(p, R, nullptr);
        // 3. chunks of board rows: project the undetected ones, keep those with a candidate in reach, replay the matching in order
        for (int r0 = 0; r0 < B.n; r0 += MREFINE_THREADS) {
            const int r = r0 + tid;
            float pr[8];
            bool keep = r < B.n && !((s_found[r >> 5] >> (r & 31)) & 1u);
            if (keep) {
                if (a.has_cam) refine_project(B.obj, r, R, p, a.cam, pr);
                else refine_transform(B.obj, r, p, pr);
                keep = refine_has_candidate(a.rp, pr, n_rej, rej, s_taken);
            }
            const unsigned m = __ballot_sync(0xffffffffu, keep);
            if (lane == 0) s_wcnt[warp] = __popc(m);
            __syncthreads();
            int pos = __popc(m & ((1u << lane) - 1u));
            for (int w = 0; w < warp; w++) pos += s_wcnt[w];
            if (keep) {
                s_surv[pos] = r;
                for (int c = 0; c < 8; c++) s_proj[pos][c] = pr[c];
            }
            if (tid == 0) {
                int ns = 0;
                for (int w = 0; w < MREFINE_THREADS / 32; w++) ns += s_wcnt[w];
                s_ns = ns;
            }
            __syncthreads();
            if (warp == 0) {
                const WarpLanes L;
                for (int s = 0; s < s_ns; s++) {
                    const int id = s_rowid[s_surv[s]];
                    float q[8];
                    const int j = refine_match(L, gray, a.W, a.H, a.P, a.dict, a.rp, id, s_proj[s], n_rej, rej, s_taken, s_warp, s_hist, q);
                    if (j < 0) continue;
                    const int n = s_n;
                    if (n >= a.max_markers || n >= FID_MAX_MARKERS) {
                        // no slot for a marker cv2 would append: stop refining this frame.  Going on without it would let later
                        // markers take the candidate this one took in cv2, and every result after it would differ from cv2's.
                        if (lane == 0) {
                            atomicOr(a.overflow, 32u);
                            s_full = 1;
                        }
                        break;
                    }
                    if (lane < 4) {
                        float xy[2] = {q[2 * lane], q[2 * lane + 1]};
                        if (a.P.corner_refine == 1) {
                            float patch[(2 * FID_SUBPIX_MAX_WIN + 3) * (2 * FID_SUBPIX_MAX_WIN + 3)];
                            refine_subpix_corner(gray, a.W, a.H, a.P, a.subpix_masks, q, lane, xy, patch);
                        }
                        corners[(size_t)n * 8 + 2 * lane] = xy[0];
                        corners[(size_t)n * 8 + 2 * lane + 1] = xy[1];
                    }
                    if (lane == 0) {
                        ids[n] = id;
                        s_taken[j] = 1;
                        a.rec_idx[(size_t)f * a.max_markers + s_nrec] = j;
                        a.rec_board[(size_t)f * a.max_markers + s_nrec] = label;
                        s_nrec++;
                        s_ntaken++;
                        s_n = n + 1;
                    }
                    __syncwarp();
                }
            }
            __syncthreads();
            if (s_full) break;
        }
    }
    __syncthreads();
    if (tid == 0) {
        a.count[f] = s_n;
        a.n_rec[f] = s_nrec;
    }
}

// ---------------------------------------------------------------------------------------------------
// ChArUco diamonds (diamond.cuh), an opt-in stage of its own after every other stage.  It reads the frame's final marker list and
// leaves it unchanged: the loop's cornerSubPix write-backs go to a copy in shared memory.
struct DiamondArgs {
    const uint8_t* src;
    size_t row_stride, frame_stride;
    int enc, W, H;
    DevParams P;
    const float* subpix_masks;  // windows 1..5 (k_finish's table)
    const float* ch_masks;      // charuco_subpix_masks
    DiamondLayout layout;
    int win_default, max_iters;  // as CharucoArgs
    double eps_sq;
    int has_cam;
    Camera cam;
    int max_markers;
    const int32_t* count;   // [F]                     the markers (k_finish, k_marker_refine, or one host list)
    const int32_t* ids;     // [F][max_markers]
    const float* corners;   // [F][max_markers][8]
    const int32_t* run;     // as BoardPoseArgs
    int family;             // the diamonds' dictionary index (read with run only)
    int32_t id_offset;      // its id_offset: pose.fiducial_id = ids[0] + id_offset
    int32_t* n_out;         // [F]
    fid_diamond* out;       // [F][FID_MAX_DIAMONDS]
};

#define DIAMOND_THREADS 128
#define DIAMOND_WARPS (DIAMOND_THREADS / 32)

// One block per frame.  The warps predict every marker's three neighbours (they depend on that marker alone), warp 0 replays the
// order-dependent loop with lane-parallel candidate screens, predicting again only markers whose corners a recovery refined, then a
// warp per diamond finds its chessboard corners (approximate pose with a camera, a lane per corner, the board check), and a thread
// per kept diamond, in loop order, solves its pose.
__global__ void __launch_bounds__(DIAMOND_THREADS) k_diamond(const DiamondArgs a) {
    __shared__ float s_wc[FID_MAX_MARKERS * 8];
    __shared__ float s_pred[FID_MAX_MARKERS * 24];
    __shared__ uint8_t s_ok[FID_MAX_MARKERS], s_dirty[FID_MAX_MARKERS], s_taken[FID_MAX_MARKERS];
    __shared__ int32_t s_dia[FID_MAX_DIAMONDS * 4], s_pos[FID_MAX_DIAMONDS];
    __shared__ float s_xy[FID_MAX_DIAMONDS * 8];
    __shared__ float s_det[DIAMOND_WARPS][32];
    __shared__ double s_mn[DIAMOND_WARPS][32];
    __shared__ DiamondLayout s_L;
    __shared__ int s_nd;
    const int f = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int n = min(a.count[f], min(a.max_markers, FID_MAX_MARKERS));
    const int32_t* ids = a.ids + (size_t)f * a.max_markers;
    const float* corners = a.corners + (size_t)f * a.max_markers * 8;
    if (a.run) family_run(a.run, f, a.family, &ids, &corners, &n);
    const FrameImg gray{a.src + (size_t)f * a.frame_stride, a.row_stride, a.enc};
    for (int c = tid; c < 8 * n; c += DIAMOND_THREADS) s_wc[c] = corners[c];
    if (tid == 0) s_L = a.layout;
    __syncthreads();
    // 1. a warp per marker: its predictions from the corners as detected
    for (int i = warp; n >= 4 && i < n; i += DIAMOND_WARPS) {
        float pr[24];
        const bool ok = diamond_predict(s_L, s_wc + 8 * i, pr);
        if (lane == 0) {
            s_ok[i] = ok;
            for (int k = 0; k < 24; k++) s_pred[24 * i + k] = pr[k];
        }
    }
    __syncthreads();
    // 2. warp 0: the loop
    if (warp == 0) {
        const int nd = diamond_assign(WarpLanes{}, gray, a.W, a.H, a.P, a.subpix_masks, s_L, n, s_wc, s_pred, s_ok, s_dirty, s_taken, s_dia);
        if (lane == 0) s_nd = nd;
    }
    __syncthreads();
    const int nd = s_nd;
    // 3. a warp per diamond: its chessboard corners
    for (int k = warp; k < nd; k += DIAMOND_WARPS) {
        const int32_t* m = s_dia + 4 * k;
        float* det = s_det[warp];
        det[lane] = s_wc[8 * m[lane >> 3] + (lane & 7)];
        __syncwarp();
        int32_t tmp[4];
        diamond_tmp_ids(ids[m[0]], tmp);
        const CharucoView B = diamond_view(s_L, tmp);
        double R[9], p[6];
        if (a.has_cam) {
            BoardPoseOut po;
            solve_board_pose(16, s_L.obj, det, s_mn[warp], a.cam, &po);
            for (int j = 0; j < 3; j++) {
                p[j] = po.rvec[j];
                p[3 + j] = po.tvec[j];
            }
            rodrigues_v2m(p, R, nullptr);
        }
        float xy[2] = {-1.f, -1.f};
        bool keep = true;
        if (lane < 4) {
            float patch[(2 * FID_CHARUCO_MAX_WIN + 3) * (2 * FID_CHARUCO_MAX_WIN + 3)];
            keep = diamond_corner(B, lane, a.has_cam != 0, R, p, a.cam, gray, a.W, a.H, det, a.ch_masks, a.win_default, a.max_iters, a.eps_sq, patch, xy);
        }
        bool all = __all_sync(0xffffffffu, keep);
        if (all && s_L.check_markers && lane < 4) keep = charuco_check_corner(B, lane, xy, 4, tmp, s_L.rows, det);
        all = __all_sync(0xffffffffu, keep);
        if (lane < 4) {
            s_xy[8 * k + 2 * diamond_slot(lane)] = xy[0];
            s_xy[8 * k + 2 * diamond_slot(lane) + 1] = xy[1];
        }
        if (lane == 0) s_pos[k] = all;
        __syncwarp();
    }
    __syncthreads();
    if (tid == 0) {
        int q = 0;
        for (int k = 0; k < nd; k++) s_pos[k] = s_pos[k] ? q++ : -1;
        a.n_out[f] = q;
    }
    __syncthreads();
    // 4. a thread per kept diamond: the record and the pose
    for (int k = tid; k < nd; k += DIAMOND_THREADS) {
        if (s_pos[k] < 0) continue;
        fid_diamond r{};
        for (int j = 0; j < 4; j++) r.ids[j] = ids[s_dia[4 * k + j]];
        for (int j = 0; j < 8; j++) r.corners[j] = s_xy[8 * k + j];
        r.pose.fiducial_id = r.ids[0] + a.id_offset;
        if (a.has_cam) {
            PoseOut po;
            solve_marker_pose(r.corners, a.cam, s_L.square_length, (double)s_L.square_length, &po);
            r.status = 1;
            r.pose.reserved = po.lm_iters;
            for (int j = 0; j < 3; j++) {
                r.pose.translation[j] = po.tvec[j];
                r.pose.rvec[j] = po.rvec[j];
            }
            for (int j = 0; j < 4; j++) r.pose.rotation[j] = po.quat[j];
            r.pose.image_error = po.image_error;
            r.pose.object_error = po.object_error;
            r.pose.fiducial_area = po.area;
        }
        a.out[(size_t)f * FID_MAX_DIAMONDS + s_pos[k]] = r;
    }
}

// ---------------------------------------------------------------------------------------------------
// Several dictionaries (fid_set_dictionaries): k_finish has written each dictionary's markers, without pose, to lists of their
// own.  k_dict_merge concatenates them in dictionary order (detectMarkersMultiDict), records each marker's dictionary index, and
// solves the pose of each marker as k_pose does for its published id (id + id_offset) and its dictionary's length; with the
// pose-hypotheses option also both planar hypotheses, as k_pose_hypotheses.  One block per frame, one thread per marker.
struct DictPose {
    int32_t id_offset;
    double len;  // the dictionary's default marker length (its own, else the call's)
};

struct DictMergeArgs {
    int n_dicts;
    size_t dict_stride;        // [n_dicts] of per-dictionary lists, dict_stride markers apart
    const int32_t* count;      // [n_dicts][F]
    const int32_t* ids;        // [n_dicts][F][max_markers]
    const float* corners;      // [n_dicts][F][max_markers][8]
    int F, max_markers;
    DictPose dp[FID_MAX_DICTIONARIES];
    int do_pose;
    Camera cam;
    int n_override;
    const int32_t* override_ids;
    const double* override_lens;
    int32_t* out_count;        // [F]
    int32_t* out_ids;          // [F][max_markers]
    float* out_corners;        // [F][max_markers][8]
    int32_t* out_dict;         // [F][max_markers]
    int32_t* out_run;          // [F][FID_MAX_DICTIONARIES + 1]: dictionary d's markers are out_run[d] .. out_run[d + 1] - 1
    fid_transform* out_tf;     // [F][max_markers]
    struct fid_pose_hypotheses* out_hyp;  // [F][max_markers] or nullptr
    Counters* counters;
};

#define DICT_MERGE_THREADS 64

__global__ void __launch_bounds__(DICT_MERGE_THREADS) k_dict_merge(const DictMergeArgs a) {
    __shared__ int s_off[FID_MAX_DICTIONARIES + 1];
    const int f = blockIdx.x;
    if (threadIdx.x == 0) {
        int total = 0;
        for (int d = 0; d < a.n_dicts; d++) {
            s_off[d] = total;
            total += a.count[(size_t)d * a.F + f];
        }
        const int cap = a.max_markers < FID_MAX_MARKERS ? a.max_markers : FID_MAX_MARKERS;
        if (total > cap) {
            atomicOr(&a.counters->overflow, 32u);
            total = cap;
        }
        s_off[a.n_dicts] = total;
        a.out_count[f] = total;
        for (int d = 0; d <= a.n_dicts; d++) a.out_run[(size_t)f * (FID_MAX_DICTIONARIES + 1) + d] = min(s_off[d], total);
    }
    __syncthreads();
    const int n = s_off[a.n_dicts];
    for (int m = threadIdx.x; m < n; m += DICT_MERGE_THREADS) {
        int d = 0;
        while (m >= s_off[d + 1]) d++;
        const size_t src = (size_t)d * a.dict_stride + (size_t)f * a.max_markers + (m - s_off[d]);
        const size_t o = (size_t)f * a.max_markers + m;
        const int id = a.ids[src];
        a.out_ids[o] = id;
        a.out_dict[o] = d;
        float* oc = a.out_corners + o * 8;
        for (int k = 0; k < 8; k++) oc[k] = a.corners[src * 8 + k];
        if (!a.do_pose) continue;
        const int pub = id + a.dp[d].id_offset;
        const double len = marker_len_of(pub, a.dp[d].len, a.n_override, a.override_ids, a.override_lens);
        PoseOut po;
        solve_marker_pose(oc, a.cam, (float)len, a.dp[d].len, &po);
        fid_transform t;
        t.fiducial_id = pub;
        t.reserved = po.lm_iters;
        for (int k = 0; k < 3; k++) {
            t.translation[k] = po.tvec[k];
            t.rvec[k] = po.rvec[k];
        }
        for (int k = 0; k < 4; k++) t.rotation[k] = po.quat[k];
        t.image_error = po.image_error;
        t.object_error = po.object_error;
        t.fiducial_area = po.area;
        a.out_tf[o] = t;
        if (a.out_hyp) {
            PoseHypOut ho;
            solve_marker_hypotheses(oc, a.cam, (float)len, po.rvec, &ho);
            pack_hypotheses(pub, ho, a.out_hyp + o);
        }
    }
}

}  // namespace fid
