// CUDA kernels, back half of the per-frame pipeline (sm_90a):
//   k_sort_group  one block per frame: clockwise fix, stable descending-perimeter order, pairwise
//                 "too close" matrix, OpenCV's order-dependent grouping                  (SURVEY A.5)
//   k_identify_first / k_identify_retry   one warp per selected candidate, one block per failed first attempt: perspective removal, Otsu, cell votes, border
//                 check, first-match dictionary search (+ close-contour retry)           (A.6, A.7)
//   k_finish      one block per frame: compaction in OpenCV's output order, cornerSubPix (A.8),
//                 solvePnP(ITERATIVE) + FiducialTransform arithmetic                     (A.9)
#pragma once
#include <cuda_runtime.h>

#include "../../include/fiducials_b200.h"
#include "common.cuh"
#include "contour_refine.cuh"
#include "identify.cuh"
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
            group_finish_lanes(L, g, qs, a.marker_size, a.border_bits, a.min_group_dist, sm_selected, sm_members, &s_members_used, sm_next, sm_head, a.fs.close_count + fo,
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
        const FrameImg gray{a.src + (size_t)f * a.frame_stride, a.row_stride, a.enc};
        const IdentifyResult r = identify_candidate(L, gray, a.W, a.H, a.fs.quads[fo + si], a.P, sm_dict, img, hist);
        __syncwarp();
        if (lane == 0) {
            if (r.id >= 0) {
                identify_write(a, fo, o, r.id, r.rotation, si);
            } else if (a.fs.close_count[fo + si] > 0) {
                a.cand_id[o] = -2;
                a.retry_list[atomicAdd(&a.counters->n_retry, 1u)] = rec;
            } else {
                a.cand_id[o] = -1;
            }
        }
    }
}

// One block per candidate whose first attempt failed.  A non-marker group of a dozen nested outlines used to cost a dozen
// identifications back to back in one warp -- the longest chain of the launch.  Here warp w tries attempts 1 + w, 1 + w + 8, ...
// concurrently; the lowest successful attempt wins, which is exactly the sequential first-success rule.
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
        const FrameImg gray{a.src + (size_t)f * a.frame_stride, a.row_stride, a.enc};
        const int nc = a.fs.close_count[fo + si], co = a.fs.close_off[fo + si];
        for (int t = 1 + warp; t <= nc; t += IDENT_WARPS) {
            if (t > *reinterpret_cast<volatile int*>(&s_best)) break;  // an earlier attempt already decoded
            const QuadF quad = a.fs.quads[fo + a.fs.close_idx[fo + co + t - 1]];
            const IdentifyResult r = identify_candidate(L, gray, a.W, a.H, quad, a.P, sm_dict, img, hist);
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
            int id = -1, rot = 0, att = 0;
            for (int w = 0; w < IDENT_WARPS; w++)
                if (s_att[w] == s_best && s_best != 0x7fffffff) {
                    id = s_id[w];
                    rot = s_rot[w];
                    att = s_att[w];
                }
            if (id >= 0)
                identify_write(a, fo, o, id, rot, a.fs.close_idx[fo + co + att - 1]);
            else
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
    // nearest larger candidate whose quad contains all four corners of i
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

}  // namespace fid
