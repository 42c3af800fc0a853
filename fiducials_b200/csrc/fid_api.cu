// C-ABI of the detector (include/fiducials_b200.h): handle management, batch orchestration on CUDA
// streams, stage timing.  No CPU fallback: every entry point that computes needs a CUDA device.
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../include/fiducials_b200.h"
#include "kernels_contour.cuh"
#include "kernels_threshold.cuh"
#include "start_prune_table.h"
#include "kernels_threshold_mma.cuh"
#include "kernels_marker.cuh"
#include "params_host.h"

using namespace fid;

#define CK(call)                                                                                       \
    do {                                                                                               \
        cudaError_t e_ = (call);                                                                       \
        if (e_ != cudaSuccess) {                                                                       \
            fprintf(stderr, "[fiducials_b200] CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); \
            return FID_ERR_CUDA;                                                                       \
        }                                                                                              \
    } while (0)

enum { ST_H2D = 0, ST_THRESH, ST_MASKS, ST_WALK, ST_EMIT, ST_APPROX, ST_GROUP, ST_IDENT, ST_SUBPIX_POSE, ST_POSE_UNUSED, ST_D2H, ST_COUNT };
enum { N_WALK_ROUNDS = FID_WALK_MAX_ROUNDS };
enum { MAX_SLOTS = 8 };

struct Slot {
    uint8_t* d_bgr = nullptr;
    uint8_t* d_gray = nullptr;
    uint32_t* d_halo = nullptr;
    StartRec* d_starts = nullptr;
    ChainRec* d_chains = nullptr;
    SegRec* d_segs = nullptr;
    WalkRec* d_queue[2] = {nullptr, nullptr};
    Pt16* d_points = nullptr;
    Counters* d_counters = nullptr;
    RawQuad* d_raw = nullptr;
    unsigned int* d_nraw = nullptr;
    FrameScratch fs{};
    int* d_nsel = nullptr;
    int* d_nrawc = nullptr;
    int* d_cand_id = nullptr;
    float* d_cand_corners = nullptr;
    int* d_cand_raw = nullptr;
    uint32_t* d_first_list = nullptr;  // work lists of the identification kernels, F * max_sel records each
    uint32_t* d_retry_list = nullptr;
    int32_t* d_out_count = nullptr;
    int32_t* d_out_ids = nullptr;
    float* d_out_corners = nullptr;
    fid_transform* d_out_tf = nullptr;
    // pinned host mirrors
    int32_t* h_out_count = nullptr;
    int32_t* h_out_ids = nullptr;
    float* h_out_corners = nullptr;
    fid_transform* h_out_tf = nullptr;
    Counters* h_counters = nullptr;
    int* h_nsel = nullptr;
    int* h_nrawc = nullptr;
    cudaEvent_t ev[ST_COUNT + 1]{};
    cudaEvent_t ev_round[N_WALK_ROUNDS + 1]{};
    cudaEvent_t done = nullptr;
    cudaEvent_t copied = nullptr;
};

struct fid_detector {
    int device = 0;
    int sm_count = 132;  // H100 SXM; replaced by the device's count in fid_create
    fid_params params{};
    DevParams P{};
    int max_w = 0, max_h = 0, max_batch = 0;
    int max_raw = FID_GROUP_MAX_RAW, close_wpr = 128, max_sel = FID_MAX_SEL, max_markers = FID_MAX_MARKERS;
    unsigned int max_starts = 0, max_chains = 0, max_points = 0, max_queue = 0, max_segs = 0;
    cudaStream_t stream = nullptr, copy_stream = nullptr;
    // one compute stream per slot (chunk in flight): the latency-bound stages of one chunk overlap the
    // issue-bound stages of the others.  FID_SLOTS (2..8, default 4)
    int n_slots = 4;
    int stagger = 0;  // FID_STAGGER bit mask, see enqueue_pipeline
    int enc = FID_ENC_BGR8, bpp = 3;  // fid_set_input_encoding
    // fid_submit_batch / fid_collect_batch: FIFO of batches in flight
    struct Pending {
        int first_slot, n_chunks, n_frames, w, h;
        int64_t launches;
        bool pose;
    } pending[MAX_SLOTS]{};
    int pend_head = 0, pend_count = 0, slots_in_use = 0, slot_next = 0;
    cudaStream_t slot_stream[MAX_SLOTS] = {};
    Slot slot[MAX_SLOTS];
    // streaming prefetch (fid_hint_next): first chunk of the next call, ping-pong
    uint8_t* d_pf[2] = {nullptr, nullptr};
    cudaEvent_t pf_done[2] = {nullptr, nullptr};
    const uint8_t* pf_host = nullptr;
    const uint8_t* hint_next = nullptr;
    int pf_idx = 0, pf_frames = 0, pf_w = 0, pf_h = 0;
    float* d_subpix_masks = nullptr;
    unsigned long long* d_dict = nullptr;  // active dictionary, kMaxDictMarkers * 4 words
    uint32_t* d_prune = nullptr;           // start_prune_table.h on the device; used when start_prune is set (FID_START_PRUNE=1, default off)
    int start_prune = 0;
    uint32_t* d_lut_prev = nullptr;
    uint32_t* d_lut_next = nullptr;
    int thresh_mode = 0;  // 0 = summed-area-table kernel (kernels_threshold.cuh, default: faster end to end), 1 = tensor-core kernel (kernels_threshold_mma.cuh; FID_THRESH=mma)
    int walk_rounds = 0;
    int walk_refill = 16, walk_pass = 16;  // persistent rounds: idle lanes that trigger a refill, steps per pass (FID_WALK_REFILL / FID_WALK_PASS)
    int emit_blocks_per_sm = 8;
    int walk_budget[FID_WALK_MAX_ROUNDS]{};
    int walk_persist[FID_WALK_MAX_ROUNDS]{};
    int32_t* d_override_ids = nullptr;
    double* d_override_lens = nullptr;
    int32_t* d_pose_ids = nullptr;
    float* d_pose_corners = nullptr;
    fid_transform* d_pose_out = nullptr;
    float stage_ms[ST_COUNT + N_WALK_ROUNDS]{};
    int64_t counters[8]{};
    cudaEvent_t t0 = nullptr, t1 = nullptr;
    // last geometry (for debug calls)
    int last_w = 0, last_h = 0, last_frames = 0;
};

static const char* kErr[] = {"ok", "invalid argument", "no usable CUDA device (this library has no CPU fallback)", "CUDA runtime error", "unsupported parameter or dictionary",
                             "capacity exceeded", "out of memory"};

extern "C" const char* fid_strerror(int status) {
    const int i = -status;
    if (i < 0 || i > 6) return "unknown status";
    return kErr[i];
}
extern "C" const char* fid_version(void) { return "0.1.0"; }

extern "C" int fid_default_params(fid_params* p) {
    if (!p) return FID_ERR_INVALID_ARG;
    default_params(p);
    return FID_OK;
}

template <class T>
static int dalloc(T** p, size_t count) {
    if (cudaMalloc((void**)p, count * sizeof(T)) != cudaSuccess) {
        cudaGetLastError();
        return FID_ERR_NO_MEMORY;
    }
    return FID_OK;
}
template <class T>
static int halloc(T** p, size_t count) {
    if (cudaMallocHost((void**)p, count * sizeof(T)) != cudaSuccess) {
        cudaGetLastError();
        return FID_ERR_NO_MEMORY;
    }
    return FID_OK;
}

static FrameGeom make_geom(const fid_detector* h, int W, int H, size_t row_stride, size_t frame_stride) {
    FrameGeom g;
    g.W = W;
    g.H = H;
    g.gray_pitch = (W + 31) / 32 * 32;
    g.bgr_row_stride = row_stride;
    g.bgr_frame_stride = frame_stride;
    g.gray_frame_stride = (size_t)g.gray_pitch * H;
    g.halo_tpr = halo_tiles_x(W);
    g.halo_tiles_y = (H + FID_HALO_T - 1) / FID_HALO_T;
    g.halo_scale_stride = halo_plane_words(W, H);
    g.halo_frame_stride = g.halo_scale_stride * h->P.n_scales;
    g.magic_tpr = (uint32_t)((0x100000000ull + (uint64_t)g.halo_tpr - 1) / (uint64_t)g.halo_tpr);
    g.magic_tiles_y = (uint32_t)((0x100000000ull + (uint64_t)g.halo_tiles_y - 1) / (uint64_t)g.halo_tiles_y);
    return g;
}

// the active dictionary -> device (n_markers x 4 rotations of 64-bit words)
static int upload_dictionary(fid_detector* h) {
    std::vector<unsigned long long> words;
    pack_dictionary(h->P, &words);
    CK(cudaMemcpy(h->d_dict, words.data(), words.size() * sizeof(unsigned long long), cudaMemcpyHostToDevice));
    return FID_OK;
}

static size_t group_smem(int max_raw) { return (size_t)max_raw * 6 * sizeof(int) + (((size_t)max_raw + 15) & ~(size_t)15) + GROUP_CLOSE_SMEM_WORDS * sizeof(uint32_t); }
static size_t ident_smem(const DevParams& P, int warps) { return (size_t)P.n_markers * 4 * 8 + (size_t)warps * 256 * 4 + (size_t)warps * FID_MAX_WARP_SIDE_SQ; }

// cuTensorMapEncodeTiled through the runtime's driver entry point (no link-time dependency on libcuda)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_tiled_fn() {
    static EncodeTiledFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = (EncodeTiledFn)p;
        cudaGetLastError();
    }
    return fn;
}
// u32 view of 3-byte-per-pixel rows: dims (3W/4, H, frames), box TM_BOXW x TM_BOXH x 1.  False when the layout cannot be described
// (then every tile takes the clamping global-load path).
static bool make_bgr_tensor_map(CUtensorMap* tm, const uint8_t* src, int W, int H, int nf, size_t row_stride, size_t frame_stride) {
    EncodeTiledFn fn = encode_tiled_fn();
    if (!fn || (W & 3) || (row_stride & 15) || (frame_stride & 15) || (reinterpret_cast<uintptr_t>(src) & 15) || 3 * W / 4 < TM_BOXW || H < TM_BOXH) return false;
    const cuuint64_t gdim[3] = {(cuuint64_t)(3 * W / 4), (cuuint64_t)H, (cuuint64_t)nf};
    const cuuint64_t gstr[2] = {(cuuint64_t)row_stride, (cuuint64_t)frame_stride};
    const cuuint32_t box[3] = {TM_BOXW, TM_BOXH, 1};
    const cuuint32_t estr[3] = {1, 1, 1};
    return fn(tm, CU_TENSOR_MAP_DATA_TYPE_UINT32, 3, const_cast<uint8_t*>(src), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
              CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

static int r_max_of(const DevParams& P) {
    int r = 1;
    for (int i = 0; i < P.n_scales; i++) r = std::max(r, P.win[i] / 2);
    return r;
}

static int configure_kernels(fid_detector* h) {
    CK(cudaFuncSetAttribute(k_threshold<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)thresh_smem_bytes(THR_FAST_R)));
    CK(cudaFuncSetAttribute(k_threshold<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)thresh_smem_bytes(FID_MAX_WIN_RADIUS)));
    CK(cudaFuncSetAttribute(k_threshold<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)thresh_smem_bytes(THR_FAST_R)));
    CK(cudaFuncSetAttribute(k_threshold<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)thresh_smem_bytes(FID_MAX_WIN_RADIUS)));
    CK(cudaFuncSetAttribute(k_threshold_mma<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TM_SMEM_BYTES));
    CK(cudaFuncSetAttribute(k_threshold_mma<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TM_SMEM_BYTES));
    CK(cudaFuncSetAttribute(k_sort_group, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)group_smem(FID_GROUP_MAX_RAW)));
    CK(cudaFuncSetAttribute(k_identify_retry, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kMaxDictMarkers * 4 * 8 + IDENT_WARPS * 256 * 4 + IDENT_WARPS * FID_MAX_WARP_SIDE_SQ)));
    CK(cudaFuncSetAttribute(k_identify_first, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kMaxDictMarkers * 4 * 8 + IDENT0_WARPS * 256 * 4 + IDENT0_WARPS * FID_MAX_WARP_SIDE_SQ)));
    return FID_OK;
}

static int alloc_slot(fid_detector* h, Slot& s) {
    const size_t F = h->max_batch;
    const int W = h->max_w, H = h->max_h;
    const size_t wpr = (W + 31) / 32, pitch = wpr * 32;
    const int S = FID_MAX_SCALES;  // params may change between frames (fid_set_params)
    int rc;
#define A(expr)                  \
    if ((rc = (expr)) != FID_OK) return rc;
    A(dalloc(&s.d_bgr, F * (size_t)W * H * 3));
    A(dalloc(&s.d_gray, F * pitch * H));
    A(dalloc(&s.d_halo, F * (size_t)S * halo_plane_words(W, H)));
    A(dalloc(&s.d_starts, (size_t)h->max_starts));
    A(dalloc(&s.d_chains, (size_t)h->max_chains));
    A(dalloc(&s.d_segs, (size_t)h->max_segs));
    A(dalloc(&s.d_queue[0], (size_t)h->max_queue));
    A(dalloc(&s.d_queue[1], (size_t)h->max_queue));
    A(dalloc(&s.d_points, (size_t)h->max_points));
    A(dalloc(&s.d_counters, 1));
    const size_t R = F * h->max_raw;
    A(dalloc(&s.d_raw, R));
    A(dalloc(&s.d_nraw, F));
    A(dalloc(&s.fs.quads_tmp, R));
    A(dalloc(&s.fs.per_tmp, R));
    A(dalloc(&s.fs.quads, R));
    A(dalloc(&s.fs.per, R));
    A(dalloc(&s.fs.close_bits, R * h->close_wpr));
    A(dalloc(&s.fs.group_id, R));
    A(dalloc(&s.fs.group_members, R));
    A(dalloc(&s.fs.next_in_group, R));
    A(dalloc(&s.fs.group_head, R));
    A(dalloc(&s.fs.group_tail, R));
    A(dalloc(&s.fs.close_count, R));
    A(dalloc(&s.fs.close_idx, R));
    A(dalloc(&s.fs.close_off, R));
    A(dalloc(&s.fs.selected, R));
    A(dalloc(&s.fs.sel_idx, R));
    A(dalloc(&s.fs.raw_of_sorted, R));
    A(dalloc(&s.d_nsel, F));
    A(dalloc(&s.d_nrawc, F));
    A(dalloc(&s.d_cand_id, F * h->max_sel));
    A(dalloc(&s.d_cand_corners, F * h->max_sel * 8));
    A(dalloc(&s.d_cand_raw, F * h->max_sel));
    A(dalloc(&s.d_first_list, F * h->max_sel));
    A(dalloc(&s.d_retry_list, F * h->max_sel));
    const size_t M = F * h->max_markers;
    A(dalloc(&s.d_out_count, F));
    A(dalloc(&s.d_out_ids, M));
    A(dalloc(&s.d_out_corners, M * 8));
    A(dalloc(&s.d_out_tf, M));
    A(halloc(&s.h_out_count, F));
    A(halloc(&s.h_out_ids, M));
    A(halloc(&s.h_out_corners, M * 8));
    A(halloc(&s.h_out_tf, M));
    A(halloc(&s.h_counters, 1));
    A(halloc(&s.h_nsel, F));
    A(halloc(&s.h_nrawc, F));
#undef A
    for (int i = 0; i <= ST_COUNT; i++) CK(cudaEventCreate(&s.ev[i]));
    for (int i = 0; i <= N_WALK_ROUNDS; i++) CK(cudaEventCreate(&s.ev_round[i]));
    CK(cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&s.copied, cudaEventDisableTiming));
    return FID_OK;
}

static void free_slot(Slot& s) {
    void* dptrs[] = {s.d_segs, s.d_halo, s.d_queue[0], s.d_queue[1], s.d_bgr,         s.d_gray,          s.d_starts,       s.d_chains,       s.d_points,      s.d_counters,
                     s.d_raw,         s.d_nraw,          s.fs.quads_tmp,    s.fs.per_tmp,     s.fs.quads,       s.fs.per,         s.fs.close_bits, s.fs.group_id,
                     s.fs.group_members, s.fs.next_in_group, s.fs.group_head, s.fs.group_tail, s.fs.close_count, s.fs.close_idx,   s.fs.close_off,  s.fs.selected,
                     s.fs.sel_idx,    s.d_nsel,          s.d_nrawc,         s.d_cand_id,      s.d_cand_corners, s.d_out_count,    s.d_out_ids,     s.d_out_corners,
                     s.d_out_tf,      s.fs.raw_of_sorted, s.d_cand_raw,     s.d_first_list,   s.d_retry_list};
    for (void* p : dptrs)
        if (p) cudaFree(p);
    void* hptrs[] = {s.h_out_count, s.h_out_ids, s.h_out_corners, s.h_out_tf, s.h_counters, s.h_nsel, s.h_nrawc};
    for (void* p : hptrs)
        if (p) cudaFreeHost(p);
    for (int i = 0; i <= ST_COUNT; i++)
        if (s.ev[i]) cudaEventDestroy(s.ev[i]);
    for (int i = 0; i <= N_WALK_ROUNDS; i++)
        if (s.ev_round[i]) cudaEventDestroy(s.ev_round[i]);
    if (s.done) cudaEventDestroy(s.done);
    if (s.copied) cudaEventDestroy(s.copied);
}

extern "C" int fid_create(const fid_params* params, int device, int max_width, int max_height, int max_batch, fid_detector** out) {
    if (!params || !out || max_width < 16 || max_height < 16 || max_batch < 1 || max_width > 16384 || max_height > 16384) return FID_ERR_INVALID_ARG;
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) {
        cudaGetLastError();
        return FID_ERR_NO_DEVICE;
    }
    if ((long long)max_batch * halo_tiles_x(max_width) * ((max_height + FID_HALO_T - 1) / FID_HALO_T) > ((1ll << FID_START_TILE_BITS) - 1)) return FID_ERR_INVALID_ARG;  // StartRec tile field (all ones = null record)
    DevParams P;
    int rc = make_dev_params(*params, &P);
    if (rc != FID_OK) return rc;
    CK(cudaSetDevice(device));
    fid_detector* h = new fid_detector();
    h->device = device;
    h->params = *params;
    h->P = P;
    h->max_w = max_width;
    h->max_h = max_height;
    h->max_batch = max_batch;
#define CKH(call)                                                                                      \
    do {                                                                                               \
        cudaError_t e_ = (call);                                                                       \
        if (e_ != cudaSuccess) {                                                                       \
            fprintf(stderr, "[fiducials_b200] CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); \
            fid_destroy(h);                                                                            \
            return FID_ERR_CUDA;                                                                       \
        }                                                                                              \
    } while (0)
    cudaDeviceProp prop;
    CKH(cudaGetDeviceProperties(&prop, device));
    h->sm_count = prop.multiProcessorCount;
    const size_t px = (size_t)max_width * max_height * max_batch;
    // Worst case measured on uniform-noise frames with the reference's 13 scales: 4.9 start cracks and
    // 3.6 in-range contour points per pixel (typical marker scenes: 0.3 and 0.4).
    h->max_starts = (unsigned int)std::min<size_t>(px * 6 + 65536, 0x7fffffffu);
    h->max_chains = (unsigned int)std::min<size_t>((size_t)max_batch * 65536, 0x7fffffffu);
    h->max_points = (unsigned int)std::min<size_t>(px * 4 + 65536, 0x7fffffffu);
    h->max_segs = h->max_chains * 4;  // two per contour + checkpoints of the long ones
    h->max_queue = h->max_starts / 8 + 65536;  // walks that survive the first 32 steps: ~3 % of the start cracks
    CKH(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    CKH(cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking));
    if (const char* e = getenv("FID_STAGGER")) h->stagger = atoi(e);
    if (const char* e = getenv("FID_THRESH")) h->thresh_mode = strcmp(e, "mma") == 0 ? 1 : 0;
    if (const char* e = getenv("FID_SLOTS")) h->n_slots = std::max(2, std::min((int)MAX_SLOTS, atoi(e)));
    for (int i = 0; i < h->n_slots; i++) CKH(cudaStreamCreateWithFlags(&h->slot_stream[i], cudaStreamNonBlocking));
    if ((rc = dalloc(&h->d_dict, (size_t)kMaxDictMarkers * 4)) != FID_OK || (rc = upload_dictionary(h)) != FID_OK || (rc = configure_kernels(h)) != FID_OK) {
        fid_destroy(h);
        return rc;
    }
    if (const char* e = getenv("FID_START_PRUNE")) h->start_prune = atoi(e) != 0;  // table stage of the start pruning: proven on the CPU
    if (h->start_prune) {                                                            // (tests/test_hostsim_contours.py), off by default
        if ((rc = dalloc(&h->d_prune, (size_t)2 * FID_START_PRUNE_WORDS)) != FID_OK) {
            fid_destroy(h);
            return rc;
        }
        CKH(cudaMemcpy(h->d_prune, kStartPruneTable, sizeof(kStartPruneTable), cudaMemcpyHostToDevice));
    }
    for (int i = 0; i < h->n_slots; i++)
        if ((rc = alloc_slot(h, h->slot[i])) != FID_OK) {
            fid_destroy(h);
            return rc;
        }
    // cornerSubPix windows 1..5 (host libm, like OpenCV)
    {
        std::vector<float> masks;
        for (int w = 1; w <= 5; w++) {
            std::vector<float> m((2 * w + 1) * (2 * w + 1));
            subpix_mask(w, m.data());
            masks.insert(masks.end(), m.begin(), m.end());
        }
        if ((rc = dalloc(&h->d_subpix_masks, masks.size())) != FID_OK) {
            fid_destroy(h);
            return rc;
        }
        CKH(cudaMemcpy(h->d_subpix_masks, masks.data(), masks.size() * sizeof(float), cudaMemcpyHostToDevice));
    }
    {   // step tables of the border walk
        std::vector<uint32_t> lp(FID_LUT_SIZE), ln(FID_LUT_SIZE);
        build_step_tables(lp.data(), ln.data());
        if ((rc = dalloc(&h->d_lut_prev, (size_t)FID_LUT_SIZE)) != FID_OK || (rc = dalloc(&h->d_lut_next, (size_t)FID_LUT_SIZE)) != FID_OK) {
            fid_destroy(h);
            return rc;
        }
        CKH(cudaMemcpy(h->d_lut_prev, lp.data(), FID_LUT_SIZE * sizeof(uint32_t), cudaMemcpyHostToDevice));
        CKH(cudaMemcpy(h->d_lut_next, ln.data(), FID_LUT_SIZE * sizeof(uint32_t), cudaMemcpyHostToDevice));
    }
    {   // walk plan: budgets per round, 'p' prefix = persistent lanes, 0 = unbounded (must be last)
        if (const char* e = getenv("FID_EMIT_BLOCKS")) h->emit_blocks_per_sm = std::max(1, atoi(e));
        if (const char* e = getenv("FID_WALK_REFILL")) h->walk_refill = std::max(1, std::min(32, atoi(e)));
        if (const char* e = getenv("FID_WALK_PASS")) h->walk_pass = std::max(2, atoi(e)) & ~1;
        const char* plan = getenv("FID_WALK_PLAN");
        if (!plan || !*plan) plan = "8,64,512,p0";
        h->walk_rounds = 0;
        const char* c = plan;
        while (*c && h->walk_rounds < FID_WALK_MAX_ROUNDS) {
            int persist = 0;
            if (*c == 'p') {
                persist = 1;
                c++;
            }
            char* end = nullptr;
            long v = strtol(c, &end, 10);
            if (end == c) break;
            h->walk_budget[h->walk_rounds] = v <= 0 ? 0x3fffffff : (int)v;
            h->walk_persist[h->walk_rounds] = persist;
            h->walk_rounds++;
            c = end;
            if (*c == ',') c++;
        }
        if (h->walk_rounds == 0 || h->walk_budget[h->walk_rounds - 1] != 0x3fffffff) {
            if (h->walk_rounds == FID_WALK_MAX_ROUNDS) h->walk_rounds--;
            h->walk_budget[h->walk_rounds] = 0x3fffffff;
            h->walk_persist[h->walk_rounds] = 1;
            h->walk_rounds++;
        }
    }
    for (int i = 0; i < 2; i++) {
        if ((rc = dalloc(&h->d_pf[i], (size_t)max_batch * max_width * max_height * 3)) != FID_OK) {
            fid_destroy(h);
            return rc;
        }
        CKH(cudaEventCreateWithFlags(&h->pf_done[i], cudaEventDisableTiming));
    }
    if ((rc = dalloc(&h->d_override_ids, 1024)) != FID_OK || (rc = dalloc(&h->d_override_lens, 1024)) != FID_OK || (rc = dalloc(&h->d_pose_ids, 4096)) != FID_OK ||
        (rc = dalloc(&h->d_pose_corners, 4096 * 8)) != FID_OK || (rc = dalloc(&h->d_pose_out, 4096)) != FID_OK) {
        fid_destroy(h);
        return rc;
    }
    *out = h;
    return FID_OK;
#undef CKH
}

extern "C" int fid_destroy(fid_detector* h) {
    if (!h) return FID_ERR_INVALID_ARG;
    cudaSetDevice(h->device);
    cudaDeviceSynchronize();
    for (int i = 0; i < MAX_SLOTS; i++) free_slot(h->slot[i]);
    void* ptrs[] = {h->d_prune, h->d_dict, h->d_pf[0], h->d_pf[1], h->d_lut_prev, h->d_lut_next, h->d_subpix_masks, h->d_override_ids, h->d_override_lens, h->d_pose_ids, h->d_pose_corners, h->d_pose_out};
    for (void* p : ptrs)
        if (p) cudaFree(p);
    for (int i = 0; i < 2; i++)
        if (h->pf_done[i]) cudaEventDestroy(h->pf_done[i]);
    if (h->t0) cudaEventDestroy(h->t0);
    if (h->t1) cudaEventDestroy(h->t1);
    if (h->stream) cudaStreamDestroy(h->stream);
    if (h->copy_stream) cudaStreamDestroy(h->copy_stream);
    for (int i = 0; i < MAX_SLOTS; i++)
        if (h->slot_stream[i]) cudaStreamDestroy(h->slot_stream[i]);
    delete h;
    return FID_OK;
}

extern "C" int fid_set_params(fid_detector* h, const fid_params* params) {
    if (!h || !params) return FID_ERR_INVALID_ARG;
    DevParams P;
    const int rc = make_dev_params(*params, &P);
    if (rc != FID_OK) return rc;
    if (h->pend_count) return FID_ERR_INVALID_ARG;  // between frames only (configCallback, aruco_detect.cpp:257-298)
    CK(cudaSetDevice(h->device));
    for (int i = 0; i < h->n_slots; i++) CK(cudaStreamSynchronize(h->slot_stream[i]));
    CK(cudaStreamSynchronize(h->stream));
    h->params = *params;
    h->P = P;
    return upload_dictionary(h);
}

static Camera make_camera(const fid_camera* c) {
    Camera cam{};
    if (c) {
        cam.fx = c->K[0];
        cam.fy = c->K[4];
        cam.cx = c->K[2];
        cam.cy = c->K[5];
        cam.k1 = c->D[0];
        cam.k2 = c->D[1];
        cam.p1 = c->D[2];
        cam.p2 = c->D[3];
        cam.k3 = c->D[4];
    }
    return cam;
}

// Launch with a per-launch scheduling priority (cudaLaunchAttributePriority).  Several chunks are in flight on separate streams;
// when SM resources free up, the block scheduler serves the pending kernel with the highest priority first.  The later a stage
// sits in a chunk's chain, the higher its priority: the latency-bound tail kernels (last walk rounds, grouping, identification,
// pose) then slip into the gaps of the issue-bound bulk kernels (threshold, first walk rounds) of younger chunks instead of
// queueing behind their thousands of blocks.  level: 0 = bulk ... 3 = tail.
static int g_prio_lo = 0, g_prio_hi = 0, g_prio_mode = -1;
template <typename... KArgs, typename... Args>
static inline void launch_prio(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, int level, Args&&... args) {
    if (g_prio_mode < 0) {
        const char* e = getenv("FID_PRIO");
        g_prio_mode = e ? atoi(e) : 1;
        cudaDeviceGetStreamPriorityRange(&g_prio_lo, &g_prio_hi);  // lo = least (numerically largest), hi = greatest
    }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributePriority;
    at[0].val.priority = g_prio_mode ? std::max(g_prio_hi, g_prio_lo - level) : g_prio_lo;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}


// Enqueue the whole pipeline for `nf` frames resident in d_bgr (geometry g) on stream `st`.
static int enqueue_pipeline(fid_detector* h, Slot& s, cudaStream_t st, int nf, const FrameGeom& g, const uint8_t* d_bgr, const fid_camera* cam, double fiducial_len,
                            int n_override, int stop_after /* -1 = all */, const Slot* prev = nullptr) {
    const DevParams& P = h->P;
    const int W = g.W, H = g.H;
    int launches = 0;
    CK(cudaMemsetAsync(s.d_counters, 0, sizeof(Counters), st));
    CK(cudaMemsetAsync(s.d_nraw, 0, sizeof(unsigned int) * nf, st));
    // stagger: a stage of this chunk starts after the same stage of the previous chunk has finished, so the
    // low-occupancy tails of one chunk (last walk round, grouping, identification, pose) run under the
    // throughput-bound stages of the other instead of under its own twin
    if (prev && (h->stagger & 1)) CK(cudaStreamWaitEvent(st, prev->ev[ST_MASKS], 0));
    CK(cudaEventRecord(s.ev[ST_THRESH], st));
    {  // threshold stage: gray + 13 adaptive thresholds -> halo tiles + start cracks
        bool fast = P.n_scales == 13;
        for (int i = 0; i < P.n_scales; i++) fast = fast && P.win[i] == 3 + 4 * i;
        if (fast && h->thresh_mode == 1) {
            // tensor-core kernel: persistent, one CTA per SM; BGR staged by TMA where the layout allows
            ThreshMmaArgs a{};
            a.src = d_bgr;
            a.enc = h->enc;
            a.bpp = h->bpp;
            a.row_stride = g.bgr_row_stride;
            a.frame_stride = g.bgr_frame_stride;
            a.halo = s.d_halo;
            a.W = W;
            a.H = H;
            a.n_frames = nf;
            a.halo_tpr = g.halo_tpr;
            a.halo_tiles_y = g.halo_tiles_y;
            a.halo_scale_stride = g.halo_scale_stride;
            a.halo_frame_stride = g.halo_frame_stride;
            a.thresh_c = P.thresh_c;
            a.tiles_x = (g.halo_tpr + THR_TILES_X - 1) / THR_TILES_X;
            a.tiles_y = (g.halo_tiles_y + THR_TILES_Y - 1) / THR_TILES_Y;
            a.starts = s.d_starts;
            a.counters = s.d_counters;
            a.max_starts = h->max_starts;
            CUtensorMap tmap;
            memset(&tmap, 0, sizeof(tmap));
            static const bool tma_off = getenv("FID_THRESH_TMA") && atoi(getenv("FID_THRESH_TMA")) == 0;  // debugging switch
            a.use_tma = (!tma_off && h->enc != FID_ENC_MONO8 && make_bgr_tensor_map(&tmap, d_bgr, W, H, nf, g.bgr_row_stride, g.bgr_frame_stride)) ? 1 : 0;
            const long long total = (long long)a.tiles_x * a.tiles_y * nf;
            const int grid = (int)std::min<long long>(total, h->sm_count);
            static const bool prof_on = getenv("FID_THRESH_PROF") && atoi(getenv("FID_THRESH_PROF")) != 0;  // debugging: per-warp wait cycles
            static long long* d_prof = nullptr;
            if (prof_on && !d_prof) cudaMalloc((void**)&d_prof, sizeof(long long) * 256 * 16 * TM_PROF_KINDS);
            a.prof = prof_on ? d_prof : nullptr;
            if (prof_on)
                k_threshold_mma<true><<<grid, TM_THREADS, TM_SMEM_BYTES, st>>>(a, tmap);
            else
                k_threshold_mma<false><<<grid, TM_THREADS, TM_SMEM_BYTES, st>>>(a, tmap);
            launches++;
            if (prof_on && stop_after == ST_THRESH) {  // fid_debug_time_threshold: print the wait profile of a few CTAs
                cudaStreamSynchronize(st);
                std::vector<long long> hp((size_t)256 * 16 * TM_PROF_KINDS);
                cudaMemcpy(hp.data(), d_prof, hp.size() * sizeof(long long), cudaMemcpyDeviceToHost);
                static int printed = 0;
                if (printed++ < 2)
                    for (int b : {0, 1, 77}) {
                        for (int w = 0; w < 16; w++) {
                            fprintf(stderr, "[thr prof] cta %3d warp %2d:", b, w);
                            for (int k = 0; k < TM_PROF_KINDS; k++) fprintf(stderr, " %8lld", hp[((size_t)b * 16 + w) * TM_PROF_KINDS + k]);
                            fprintf(stderr, "\n");
                        }
                    }
            }
        } else {
            ThreshArgs a{};
            a.src = d_bgr;
            a.src_row_stride = g.bgr_row_stride;
            a.src_frame_stride = g.bgr_frame_stride;
            a.enc = h->enc;
            a.aligned4 = (W % 4 == 0) && (g.bgr_row_stride % 4 == 0) && (g.bgr_frame_stride % 4 == 0) && ((uintptr_t)d_bgr % 4 == 0);
            a.halo = s.d_halo;
            a.W = W;
            a.H = H;
            a.n_frames = nf;
            a.halo_tpr = g.halo_tpr;
            a.halo_tiles_y = g.halo_tiles_y;
            a.halo_scale_stride = g.halo_scale_stride;
            a.halo_frame_stride = g.halo_frame_stride;
            a.n_scales = P.n_scales;
            a.r_max = r_max_of(P);
            a.thresh_c = P.thresh_c;
            a.starts = s.d_starts;
            a.counters = s.d_counters;
            a.max_starts = h->max_starts;
            a.prune = h->start_prune ? h->d_prune : nullptr;
            for (int i = 0; i < P.n_scales; i++) a.win[i] = P.win[i];
            dim3 grid((g.halo_tpr + THR_TILES_X - 1) / THR_TILES_X, (g.halo_tiles_y + THR_TILES_Y - 1) / THR_TILES_Y, nf);
            if (a.prune) {
                if (fast)
                    launch_prio(k_threshold<true, true>, grid, dim3(THR_THREADS), thresh_smem_bytes(THR_FAST_R), st, 0, a);
                else
                    launch_prio(k_threshold<false, true>, grid, dim3(THR_THREADS), thresh_smem_bytes(a.r_max), st, 0, a);
            } else if (fast) {
                launch_prio(k_threshold<true>, grid, dim3(THR_THREADS), thresh_smem_bytes(THR_FAST_R), st, 0, a);
            } else {
                launch_prio(k_threshold<false>, grid, dim3(THR_THREADS), thresh_smem_bytes(a.r_max), st, 0, a);
            }
            launches++;
        }
    }
    CK(cudaEventRecord(s.ev[ST_MASKS], st));
    if (stop_after == ST_THRESH) return FID_OK;
    CK(cudaEventRecord(s.ev[ST_WALK], st));
    if (prev && (h->stagger & 2)) CK(cudaStreamWaitEvent(st, prev->ev[ST_EMIT], 0));
    const int mx = W > H ? W : H;
    const int min_len = (int)(P.min_perimeter_rate * mx), max_len = (int)(P.max_perimeter_rate * mx);
    {  // walk, in rounds of growing budget
        WalkArgs a{};
        a.halo = s.d_halo;
        a.lut_prev = h->d_lut_prev;
        a.lut_next = h->d_lut_next;
        a.starts = s.d_starts;
        a.chains = s.d_chains;
        a.segs = s.d_segs;
        a.max_segs = h->max_segs;
        a.counters = s.d_counters;
        a.max_starts = h->max_starts;
        a.max_chains = h->max_chains;
        a.max_points = h->max_points;
        a.max_queue = h->max_queue;
        a.g = g;
        a.min_len = min_len;
        a.max_len = max_len;
        for (int r = 0; r < N_WALK_ROUNDS; r++) {
            CK(cudaEventRecord(s.ev_round[r], st));
            if (r >= h->walk_rounds) continue;
            a.round = r;
            a.budget = h->walk_budget[r];
            a.persistent = h->walk_persist[r];
            a.q_in = r > 0 ? s.d_queue[(r - 1) & 1] : nullptr;
            a.q_out = s.d_queue[r & 1];
            a.chunk = r == 0 ? 256u : 32u;
            a.refill_min = h->walk_refill;
            a.pass_steps = h->walk_pass;
            static const int wb2 = getenv("FID_WALK_BLOCKS_R2") ? atoi(getenv("FID_WALK_BLOCKS_R2")) : 4, wb3 = getenv("FID_WALK_BLOCKS_R3") ? atoi(getenv("FID_WALK_BLOCKS_R3")) : 4;
            const int blocks = r == 0 ? h->sm_count * 8 : (r == 1 ? h->sm_count * 8 : h->sm_count * (r == 2 ? wb2 : wb3));
            launch_prio(k_walk, dim3(blocks), dim3(256), 0, st, r == 0 ? 1 : (r == 1 ? 2 : 3), a);
            launches++;
        }
        CK(cudaEventRecord(s.ev_round[N_WALK_ROUNDS], st));
    }
    CK(cudaEventRecord(s.ev[ST_EMIT], st));
    {  // emit
        EmitArgs a{};
        a.halo = s.d_halo;
        a.lut_prev = h->d_lut_prev;
        a.lut_next = h->d_lut_next;
        a.segs = s.d_segs;
        a.points = s.d_points;
        a.counters = s.d_counters;
        a.work_counter = &s.d_counters->emit_work;
        a.max_segs = h->max_segs;
        a.g = g;
        launch_prio(k_emit, dim3(h->sm_count * h->emit_blocks_per_sm), dim3(64), 0, st, 3, a);
        launches++;
    }
    CK(cudaEventRecord(s.ev[ST_APPROX], st));
    {  // approx
        ApproxArgs a{};
        a.chains = s.d_chains;
        a.points = s.d_points;
        a.counters = s.d_counters;
        a.raw = s.d_raw;
        a.n_raw = s.d_nraw;
        a.counters_rw = s.d_counters;
        a.max_chains = h->max_chains;
        a.max_raw = h->max_raw;
        a.W = W;
        a.H = H;
        a.poly_accuracy_rate = P.poly_accuracy_rate;
        a.min_corner_dist_rate = P.min_corner_dist_rate;
        launch_prio(k_approx_warp, dim3(h->sm_count * 8), dim3(APPROX_THREADS), 0, st, 3, a);
        launches++;
        launch_prio(k_approx, dim3(h->sm_count * 4), dim3(APPROX_THREADS), 0, st, 3, a);
        launches++;
    }
    CK(cudaEventRecord(s.ev[ST_GROUP], st));
    if (stop_after == ST_APPROX) return FID_OK;
    {  // sort + group
        GroupArgs a{};
        a.raw = s.d_raw;
        a.n_raw = s.d_nraw;
        a.fs = s.fs;
        a.n_sel = s.d_nsel;
        a.n_raw_clamped = s.d_nrawc;
        a.max_raw = h->max_raw;
        a.close_wpr = h->close_wpr;
        a.max_sel = h->max_sel;
        a.marker_size = P.marker_size;
        a.border_bits = P.marker_border_bits;
        a.min_marker_dist_rate = (float)P.min_marker_dist_rate;
        a.min_group_dist = (float)P.min_group_dist;
        a.W = W;
        a.H = H;
        a.min_dist_to_border = P.min_dist_to_border;
        a.counters = s.d_counters;
        a.first_list = s.d_first_list;
        static const int group_prof = getenv("FID_GROUP_PROF") ? atoi(getenv("FID_GROUP_PROF")) : 0;
        a.prof = group_prof;
        launch_prio(k_sort_group, dim3(nf), dim3(GROUP_THREADS), group_smem(h->max_raw), st, 4, a);
        launches++;
    }
    CK(cudaEventRecord(s.ev[ST_IDENT], st));
    {  // identify
        IdentifyArgs a{};
        a.src = d_bgr;
        a.row_stride = g.bgr_row_stride;
        a.frame_stride = g.bgr_frame_stride;
        a.enc = h->enc;
        a.W = W;
        a.H = H;
        a.fs = s.fs;
        a.n_sel = s.d_nsel;
        a.max_raw = h->max_raw;
        a.max_sel = h->max_sel;
        a.P = P;
        a.dict = h->d_dict;
        a.cand_id = s.d_cand_id;
        a.cand_corners = s.d_cand_corners;
        a.cand_raw = s.d_cand_raw;
        a.first_list = s.d_first_list;
        a.retry_list = s.d_retry_list;
        a.counters = s.d_counters;
        // fixed grids over work lists: a grid of one block per (frame, candidate slot) is 32 768 blocks of which 1 500 have work
        launch_prio(k_identify_first, dim3(h->sm_count * 4), dim3(IDENT0_WARPS * 32), ident_smem(P, IDENT0_WARPS), st, 4, a);
        launch_prio(k_identify_retry, dim3(h->sm_count * 2), dim3(IDENT_WARPS * 32), ident_smem(P, IDENT_WARPS), st, 4, a);
        launches += 2;
    }
    CK(cudaEventRecord(s.ev[ST_SUBPIX_POSE], st));
    if (P.corner_refine == 2) {  // CORNER_REFINE_CONTOUR: rewrite the decoded candidates' corners before the output stage
        ContourRefineArgs a{};
        a.n_sel = s.d_nsel;
        a.cand_id = s.d_cand_id;
        a.cand_raw = s.d_cand_raw;
        a.cand_corners = s.d_cand_corners;
        a.raw = s.d_raw;
        a.points = s.d_points;
        a.max_raw = h->max_raw;
        a.max_sel = h->max_sel;
        launch_prio(k_contour_refine, dim3(h->max_sel, nf), dim3(CREFINE_THREADS), 0, st, 5, a);
        launches++;
    }
    {  // finish
        FinishArgs a{};
        a.src = d_bgr;
        a.row_stride = g.bgr_row_stride;
        a.frame_stride = g.bgr_frame_stride;
        a.enc = h->enc;
        a.W = W;
        a.H = H;
        a.n_sel = s.d_nsel;
        a.cand_id = s.d_cand_id;
        a.cand_corners = s.d_cand_corners;
        a.fs = s.fs;
        a.max_raw = h->max_raw;
        a.max_sel = h->max_sel;
        a.max_markers = h->max_markers;
        a.P = P;
        a.subpix_masks = h->d_subpix_masks;
        a.do_pose = cam ? 1 : 0;
        a.cam = make_camera(cam);
        a.fiducial_len = fiducial_len;
        a.n_override = n_override;
        a.override_ids = h->d_override_ids;
        a.override_lens = h->d_override_lens;
        a.out_count = s.d_out_count;
        a.out_ids = s.d_out_ids;
        a.out_corners = s.d_out_corners;
        a.out_tf = s.d_out_tf;
        a.counters = s.d_counters;
        launch_prio(k_finish, dim3(nf), dim3(FINISH_THREADS), 0, st, 5, a);
        launches++;
    }
    CK(cudaEventRecord(s.ev[ST_D2H], st));
    h->counters[6] += launches;
    CK(cudaGetLastError());
    return FID_OK;
}

static int enqueue_d2h(fid_detector* h, Slot& s, cudaStream_t st, int nf, bool with_pose) {
    const size_t M = (size_t)nf * h->max_markers;
    CK(cudaMemcpyAsync(s.h_out_count, s.d_out_count, sizeof(int32_t) * nf, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(s.h_out_ids, s.d_out_ids, sizeof(int32_t) * M, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(s.h_out_corners, s.d_out_corners, sizeof(float) * 8 * M, cudaMemcpyDeviceToHost, st));
    if (with_pose) CK(cudaMemcpyAsync(s.h_out_tf, s.d_out_tf, sizeof(fid_transform) * M, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(s.h_counters, s.d_counters, sizeof(Counters), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(s.h_nsel, s.d_nsel, sizeof(int) * nf, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(s.h_nrawc, s.d_nrawc, sizeof(int) * nf, cudaMemcpyDeviceToHost, st));
    CK(cudaEventRecord(s.ev[ST_COUNT], st));
    CK(cudaEventRecord(s.done, st));
    return FID_OK;
}

static int collect(fid_detector* h, Slot& s, int nf, int max_markers, int32_t* counts, int32_t* ids, float* corners, fid_transform* tfs, bool first_chunk) {
    CK(cudaEventSynchronize(s.done));
    int status = FID_OK;
    if (s.h_counters->overflow) status = FID_ERR_CAPACITY;
    for (int f = 0; f < nf; f++) {
        int n = s.h_out_count[f];
        if (n > max_markers) {
            n = max_markers;
            status = FID_ERR_CAPACITY;
        }
        counts[f] = n;
        if (ids) memcpy(ids + (size_t)f * max_markers, s.h_out_ids + (size_t)f * h->max_markers, sizeof(int32_t) * n);
        if (corners) memcpy(corners + (size_t)f * max_markers * 8, s.h_out_corners + (size_t)f * h->max_markers * 8, sizeof(float) * 8 * n);
        if (tfs) memcpy(tfs + (size_t)f * max_markers, s.h_out_tf + (size_t)f * h->max_markers, sizeof(fid_transform) * n);
    }
    // statistics
    float ms = 0;
    static const int order[] = {ST_THRESH, ST_MASKS, ST_WALK, ST_EMIT, ST_APPROX, ST_GROUP, ST_IDENT, ST_SUBPIX_POSE, ST_D2H, ST_COUNT};
    if (first_chunk) {
        for (int i = 0; i < ST_COUNT + N_WALK_ROUNDS; i++) h->stage_ms[i] = 0;
        for (int i = 0; i < 6; i++) h->counters[i] = 0;
    }
    for (int i = 0; i + 1 < (int)(sizeof(order) / sizeof(order[0])); i++) {
        if (cudaEventElapsedTime(&ms, s.ev[order[i]], s.ev[order[i + 1]]) == cudaSuccess) {
            const int dst = order[i] == ST_D2H ? ST_D2H : order[i];
            h->stage_ms[dst] += ms;
        } else {
            cudaGetLastError();
        }
    }
    for (int r = 0; r < N_WALK_ROUNDS; r++) {
        if (cudaEventElapsedTime(&ms, s.ev_round[r], s.ev_round[r + 1]) == cudaSuccess)
            h->stage_ms[ST_COUNT + r] += ms;
        else
            cudaGetLastError();
    }
    h->counters[0] += (int64_t)s.h_counters->n_starts[0] + s.h_counters->n_starts[1];
    h->counters[1] += s.h_counters->n_chains;
    h->counters[2] += s.h_counters->n_points;
    for (int f = 0; f < nf; f++) {
        h->counters[3] += s.h_nrawc[f];
        h->counters[4] += s.h_nsel[f];
        h->counters[5] += s.h_out_count[f];
    }
    return status;
}

static int upload_overrides(fid_detector* h, int n_override, const int32_t* ids, const double* lens) {
    if (n_override < 0 || n_override > 1024 || (n_override > 0 && (!ids || !lens))) return FID_ERR_INVALID_ARG;
    if (n_override > 0) {
        CK(cudaMemcpyAsync(h->d_override_ids, ids, sizeof(int32_t) * n_override, cudaMemcpyHostToDevice, h->stream));
        CK(cudaMemcpyAsync(h->d_override_lens, lens, sizeof(double) * n_override, cudaMemcpyHostToDevice, h->stream));
        CK(cudaStreamSynchronize(h->stream));  // the slot streams read them
    }
    return FID_OK;
}

extern "C" int fid_detect_pose_batch(fid_detector* h, int n_frames, const uint8_t* bgr, int bgr_on_device, int width, int height, size_t row_stride, size_t frame_stride,
                                     const fid_camera* cam, double fiducial_len, int n_override, const int32_t* override_ids, const double* override_lens,
                                     int max_markers, int32_t* counts, int32_t* ids, float* corners, fid_transform* transforms) {
    if (!h || !bgr || !counts || n_frames < 0 || width < 16 || height < 16 || width > h->max_w || height > h->max_h || max_markers < 0) return FID_ERR_INVALID_ARG;
    if (row_stride < (size_t)width * h->bpp || frame_stride < row_stride * (size_t)height) return FID_ERR_INVALID_ARG;
    if (cam && !(fiducial_len > 0)) return FID_ERR_INVALID_ARG;
    if (h->pend_count) return FID_ERR_INVALID_ARG;  // batches submitted with fid_submit_batch are still in flight
    CK(cudaSetDevice(h->device));
    int rc = upload_overrides(h, n_override, override_ids, override_lens);
    if (rc != FID_OK) return rc;
    h->last_w = width;
    h->last_h = height;
    int status = FID_OK;
    const int B = h->max_batch;
    const int n_chunks = (n_frames + B - 1) / B;
    h->counters[6] = 0;
    h->stage_ms[ST_H2D] = 0;
    // software pipeline over chunks: up to n_slots chunks in flight, each on its own stream; results of
    // chunk c are collected n_slots-1 chunks later
    const int NS = h->n_slots;
    for (int c = 0; c < n_chunks + NS - 1; c++) {
        if (c < n_chunks) {
            Slot& s = h->slot[c % NS];
            cudaStream_t cst = h->slot_stream[c % NS];
            const int nf = std::min(B, n_frames - c * B);
            const uint8_t* src = bgr + (size_t)c * B * frame_stride;
            const uint8_t* d_in;
            FrameGeom g;
            const bool contiguous = row_stride == (size_t)width * h->bpp && frame_stride == row_stride * height;
            if (bgr_on_device) {
                d_in = src;
                g = make_geom(h, width, height, row_stride, frame_stride);
            } else if (c == 0 && h->pf_host == bgr && h->pf_frames == nf && h->pf_w == width && h->pf_h == height && contiguous) {
                // first chunk was uploaded in the background during the previous call (fid_hint_next)
                CK(cudaStreamWaitEvent(h->slot_stream[0], h->pf_done[h->pf_idx], 0));
                d_in = h->d_pf[h->pf_idx];
                g = make_geom(h, width, height, (size_t)width * h->bpp, (size_t)width * h->bpp * height);
                h->pf_host = nullptr;
            } else {
                // slot reuse: its previous results must have been collected (done below) before overwrite
                if (row_stride == (size_t)width * h->bpp && frame_stride == row_stride * height) {
                    CK(cudaMemcpyAsync(s.d_bgr, src, (size_t)nf * frame_stride, cudaMemcpyHostToDevice, h->copy_stream));
                } else {
                    for (int f = 0; f < nf; f++)
                        CK(cudaMemcpy2DAsync(s.d_bgr + (size_t)f * width * h->bpp * height, (size_t)width * h->bpp, src + (size_t)f * frame_stride, row_stride, (size_t)width * h->bpp, height,
                                             cudaMemcpyHostToDevice, h->copy_stream));
                }
                CK(cudaEventRecord(s.copied, h->copy_stream));
                CK(cudaStreamWaitEvent(cst, s.copied, 0));
                d_in = s.d_bgr;
                g = make_geom(h, width, height, (size_t)width * h->bpp, (size_t)width * h->bpp * height);
            }
            if (c == n_chunks - 1 && h->hint_next && !bgr_on_device && contiguous) {
                // all uploads of this call are queued: start on the first chunk of the next call
                const int nf0 = std::min(B, n_frames);
                const int idx = h->pf_idx ^ 1;
                CK(cudaMemcpyAsync(h->d_pf[idx], h->hint_next, (size_t)nf0 * frame_stride, cudaMemcpyHostToDevice, h->copy_stream));
                CK(cudaEventRecord(h->pf_done[idx], h->copy_stream));
                h->pf_idx = idx;
                h->pf_host = h->hint_next;
                h->pf_frames = nf0;
                h->pf_w = width;
                h->pf_h = height;
                h->hint_next = nullptr;
            }
            rc = enqueue_pipeline(h, s, cst, nf, g, d_in, cam, fiducial_len, n_override, -1, c > 0 ? &h->slot[(c - 1) % NS] : nullptr);
            if (rc != FID_OK) return rc;
            rc = enqueue_d2h(h, s, cst, nf, cam != nullptr);
            if (rc != FID_OK) return rc;
            h->last_frames = nf;
        }
        if (c >= NS - 1) {
            const int pc = c - (NS - 1);
            Slot& s = h->slot[pc % NS];
            const int nf = std::min(B, n_frames - pc * B);
            rc = collect(h, s, nf, max_markers, counts + (size_t)pc * B, ids ? ids + (size_t)pc * B * max_markers : nullptr,
                         corners ? corners + (size_t)pc * B * max_markers * 8 : nullptr, (transforms && cam) ? transforms + (size_t)pc * B * max_markers : nullptr, pc == 0);
            if (rc != FID_OK) status = rc;
        }
    }
    return status;
}

extern "C" int fid_submit_batch(fid_detector* h, int n_frames, const uint8_t* bgr, int bgr_on_device, int width, int height, size_t row_stride, size_t frame_stride,
                                const fid_camera* cam, double fiducial_len, int n_override, const int32_t* override_ids, const double* override_lens) {
    if (!h || !bgr || n_frames <= 0 || width < 16 || height < 16 || width > h->max_w || height > h->max_h) return FID_ERR_INVALID_ARG;
    if (row_stride < (size_t)width * h->bpp || frame_stride < row_stride * (size_t)height) return FID_ERR_INVALID_ARG;
    if (cam && !(fiducial_len > 0)) return FID_ERR_INVALID_ARG;
    const int B = h->max_batch, NS = h->n_slots;
    const int n_chunks = (n_frames + B - 1) / B;
    if (n_chunks > NS - h->slots_in_use || h->pend_count >= MAX_SLOTS) return FID_ERR_CAPACITY;
    CK(cudaSetDevice(h->device));
    if (n_override > 0)  // the override table is shared: batches in flight must be done with it
        for (int i = 0; i < NS; i++) CK(cudaStreamSynchronize(h->slot_stream[i]));
    int rc = upload_overrides(h, n_override, override_ids, override_lens);
    if (rc != FID_OK) return rc;
    h->last_w = width;
    h->last_h = height;
    const bool contiguous = row_stride == (size_t)width * h->bpp && frame_stride == row_stride * height;
    const int first = h->slot_next;
    h->counters[6] = 0;
    for (int c = 0; c < n_chunks; c++) {
        const int si = (first + c) % NS;
        Slot& s = h->slot[si];
        cudaStream_t cst = h->slot_stream[si];
        const int nf = std::min(B, n_frames - c * B);
        const uint8_t* src = bgr + (size_t)c * B * frame_stride;
        const uint8_t* d_in;
        FrameGeom g;
        if (bgr_on_device) {
            d_in = src;
            g = make_geom(h, width, height, row_stride, frame_stride);
        } else {
            if (contiguous) {
                CK(cudaMemcpyAsync(s.d_bgr, src, (size_t)nf * frame_stride, cudaMemcpyHostToDevice, h->copy_stream));
            } else {
                for (int f = 0; f < nf; f++)
                    CK(cudaMemcpy2DAsync(s.d_bgr + (size_t)f * width * h->bpp * height, (size_t)width * h->bpp, src + (size_t)f * frame_stride, row_stride, (size_t)width * h->bpp, height,
                                         cudaMemcpyHostToDevice, h->copy_stream));
            }
            CK(cudaEventRecord(s.copied, h->copy_stream));
            CK(cudaStreamWaitEvent(cst, s.copied, 0));
            d_in = s.d_bgr;
            g = make_geom(h, width, height, (size_t)width * h->bpp, (size_t)width * h->bpp * height);
        }
        const Slot* prev = (h->slots_in_use + c) > 0 ? &h->slot[(si + NS - 1) % NS] : nullptr;
        rc = enqueue_pipeline(h, s, cst, nf, g, d_in, cam, fiducial_len, n_override, -1, prev);
        if (rc != FID_OK) return rc;
        rc = enqueue_d2h(h, s, cst, nf, cam != nullptr);
        if (rc != FID_OK) return rc;
        h->last_frames = nf;
    }
    fid_detector::Pending& pb = h->pending[(h->pend_head + h->pend_count) % MAX_SLOTS];
    pb.first_slot = first;
    pb.n_chunks = n_chunks;
    pb.n_frames = n_frames;
    pb.w = width;
    pb.h = height;
    pb.pose = cam != nullptr;
    pb.launches = h->counters[6];
    h->pend_count++;
    h->slots_in_use += n_chunks;
    h->slot_next = (first + n_chunks) % NS;
    return FID_OK;
}

extern "C" int fid_collect_batch(fid_detector* h, int max_markers, int32_t* counts, int32_t* ids, float* corners, fid_transform* transforms) {
    if (!h || !counts || max_markers < 0 || h->pend_count == 0) return FID_ERR_INVALID_ARG;
    CK(cudaSetDevice(h->device));
    const fid_detector::Pending pb = h->pending[h->pend_head];
    const int B = h->max_batch, NS = h->n_slots;
    int status = FID_OK;
    h->counters[6] = pb.launches;
    h->stage_ms[ST_H2D] = 0;
    for (int c = 0; c < pb.n_chunks; c++) {
        Slot& s = h->slot[(pb.first_slot + c) % NS];
        const int nf = std::min(B, pb.n_frames - c * B);
        const int rc = collect(h, s, nf, max_markers, counts + (size_t)c * B, ids ? ids + (size_t)c * B * max_markers : nullptr,
                               corners ? corners + (size_t)c * B * max_markers * 8 : nullptr, (transforms && pb.pose) ? transforms + (size_t)c * B * max_markers : nullptr, c == 0);
        if (rc != FID_OK) status = rc;
    }
    h->pend_head = (h->pend_head + 1) % MAX_SLOTS;
    h->pend_count--;
    h->slots_in_use -= pb.n_chunks;
    return status;
}

extern "C" int fid_detect(fid_detector* h, const uint8_t* bgr, int width, int height, size_t stride, int max_markers, int* n, int32_t* ids, float* corners) {
    if (!n) return FID_ERR_INVALID_ARG;
    int32_t count = 0;
    const int rc = fid_detect_pose_batch(h, 1, bgr, 0, width, height, stride, stride * (size_t)height, nullptr, 0.0, 0, nullptr, nullptr, max_markers, &count, ids, corners, nullptr);
    *n = count;
    return rc;
}

extern "C" int fid_pose(fid_detector* h, int n, const int32_t* ids, const float* corners, const fid_camera* cam, double fiducial_len, int n_override,
                        const int32_t* override_ids, const double* override_lens, fid_transform* out) {
    if (!h || n < 0 || n > 4096 || !cam || !(fiducial_len > 0) || (n > 0 && (!ids || !corners || !out))) return FID_ERR_INVALID_ARG;
    if (h->pend_count) return FID_ERR_INVALID_ARG;  // batches in flight read the shared override table
    if (n == 0) return FID_OK;
    CK(cudaSetDevice(h->device));
    int rc = upload_overrides(h, n_override, override_ids, override_lens);
    if (rc != FID_OK) return rc;
    CK(cudaMemcpyAsync(h->d_pose_ids, ids, sizeof(int32_t) * n, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(h->d_pose_corners, corners, sizeof(float) * 8 * n, cudaMemcpyHostToDevice, h->stream));
    PoseArgs a{};
    a.n = n;
    a.ids = h->d_pose_ids;
    a.corners = h->d_pose_corners;
    a.cam = make_camera(cam);
    a.fiducial_len = fiducial_len;
    a.n_override = n_override;
    a.override_ids = h->d_override_ids;
    a.override_lens = h->d_override_lens;
    a.out = h->d_pose_out;
    k_pose<<<(n + 63) / 64, 64, 0, h->stream>>>(a);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(out, h->d_pose_out, sizeof(fid_transform) * n, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return FID_OK;
}

extern "C" int fid_set_input_encoding(fid_detector* h, int encoding) {
    if (!h || h->pend_count) return FID_ERR_INVALID_ARG;
    if (encoding != FID_ENC_BGR8 && encoding != FID_ENC_RGB8 && encoding != FID_ENC_MONO8) return FID_ERR_UNSUPPORTED;
    h->enc = encoding;
    h->bpp = encoding == FID_ENC_MONO8 ? 1 : 3;
    h->pf_host = nullptr;  // a prefetched chunk was laid out for the old encoding
    h->hint_next = nullptr;
    return FID_OK;
}

extern "C" int fid_hint_next(fid_detector* h, const uint8_t* next_bgr) {
    if (!h) return FID_ERR_INVALID_ARG;
    h->hint_next = next_bgr;
    return FID_OK;
}

extern "C" int fid_timer_start(fid_detector* h) {
    if (!h) return FID_ERR_INVALID_ARG;
    CK(cudaSetDevice(h->device));
    if (!h->t0) {
        CK(cudaEventCreate(&h->t0));
        CK(cudaEventCreate(&h->t1));
    }
    CK(cudaStreamSynchronize(h->copy_stream));
    for (int i = 0; i < h->n_slots; i++) CK(cudaStreamSynchronize(h->slot_stream[i]));
    CK(cudaStreamSynchronize(h->stream));
    CK(cudaEventRecord(h->t0, h->stream));
    return FID_OK;
}
extern "C" int fid_timer_stop(fid_detector* h, float* elapsed_ms) {
    if (!h || !elapsed_ms || !h->t0) return FID_ERR_INVALID_ARG;
    CK(cudaSetDevice(h->device));
    CK(cudaStreamSynchronize(h->copy_stream));
    for (int i = 0; i < h->n_slots; i++) CK(cudaStreamSynchronize(h->slot_stream[i]));
    CK(cudaEventRecord(h->t1, h->stream));
    CK(cudaEventSynchronize(h->t1));
    CK(cudaEventElapsedTime(elapsed_ms, h->t0, h->t1));
    return FID_OK;
}

extern "C" int fid_host_alloc(size_t bytes, void** out) {
    if (!out) return FID_ERR_INVALID_ARG;
    if (cudaMallocHost(out, bytes) != cudaSuccess) {
        cudaGetLastError();
        return FID_ERR_NO_MEMORY;
    }
    return FID_OK;
}
extern "C" int fid_host_free(void* p) {
    if (p) cudaFreeHost(p);
    return FID_OK;
}
extern "C" int fid_device_alloc(fid_detector* h, size_t bytes, void** out) {
    if (!h || !out) return FID_ERR_INVALID_ARG;
    CK(cudaSetDevice(h->device));
    if (cudaMalloc(out, bytes) != cudaSuccess) {
        cudaGetLastError();
        return FID_ERR_NO_MEMORY;
    }
    return FID_OK;
}
extern "C" int fid_device_free(fid_detector* h, void* p) {
    if (!h) return FID_ERR_INVALID_ARG;
    CK(cudaSetDevice(h->device));
    if (p) cudaFree(p);
    return FID_OK;
}
extern "C" int fid_memcpy_h2d(fid_detector* h, void* dst_device, const void* src_host, size_t bytes) {
    if (!h || !dst_device || !src_host) return FID_ERR_INVALID_ARG;
    CK(cudaSetDevice(h->device));
    CK(cudaMemcpy(dst_device, src_host, bytes, cudaMemcpyHostToDevice));
    return FID_OK;
}

extern "C" int fid_debug_threshold(fid_detector* h, const uint8_t* bgr, int width, int height, size_t stride, uint8_t* gray, uint8_t* planes, int* n_scales) {
    if (!h || !bgr || width < 16 || height < 16 || width > h->max_w || height > h->max_h || stride < (size_t)width * h->bpp) return FID_ERR_INVALID_ARG;
    if (h->pend_count) return FID_ERR_INVALID_ARG;  // slot 0 may belong to a batch in flight
    CK(cudaSetDevice(h->device));
    Slot& s = h->slot[0];
    CK(cudaMemcpy2DAsync(s.d_bgr, (size_t)width * h->bpp, bgr, stride, (size_t)width * h->bpp, height, cudaMemcpyHostToDevice, h->stream));
    const FrameGeom g = make_geom(h, width, height, (size_t)width * h->bpp, (size_t)width * h->bpp * height);
    const int rc = enqueue_pipeline(h, s, h->stream, 1, g, s.d_bgr, nullptr, 0.0, 0, ST_THRESH);
    if (rc != FID_OK) return rc;
    if (gray) {  // the tensor-core threshold kernel keeps the gray tile on chip: produce the plane for the caller
        GrayArgs ga{};
        ga.bgr = s.d_bgr;
        ga.gray = s.d_gray;
        ga.W = width;
        ga.H = height;
        ga.n_frames = 1;
        ga.bgr_row_stride = g.bgr_row_stride;
        ga.bgr_frame_stride = g.bgr_frame_stride;
        ga.gray_pitch = g.gray_pitch;
        ga.gray_frame_stride = g.gray_frame_stride;
        ga.enc = h->enc;
        const long long gq = (long long)height * ((width + 3) / 4);
        k_gray<<<(unsigned int)((gq + 255) / 256), 256, 0, h->stream>>>(ga);
        CK(cudaGetLastError());
    }
    CK(cudaStreamSynchronize(h->stream));
    if (gray) CK(cudaMemcpy2D(gray, width, s.d_gray, g.gray_pitch, width, height, cudaMemcpyDeviceToHost));
    if (planes) {
        std::vector<uint32_t> bits((size_t)h->P.n_scales * g.halo_scale_stride);
        CK(cudaMemcpy(bits.data(), s.d_halo, bits.size() * 4, cudaMemcpyDeviceToHost));
        for (int sc = 0; sc < h->P.n_scales; sc++)
            for (int y = 0; y < height; y++)
                for (int x = 0; x < width; x++) {
                    const int tx = x / FID_HALO_T, ty = y / FID_HALO_T;
                    const uint32_t wv = bits[(size_t)sc * g.halo_scale_stride + ((size_t)ty * g.halo_tpr + tx) * 32 + (y - FID_HALO_T * ty + 1)];
                    planes[((size_t)sc * height + y) * width + x] = (wv >> (x - FID_HALO_T * tx + 1)) & 1u;
                }
    }
    if (n_scales) *n_scales = h->P.n_scales;
    return FID_OK;
}

extern "C" int fid_debug_time_threshold(fid_detector* h, int n_frames, const uint8_t* bgr_device, int width, int height, size_t row_stride, size_t frame_stride, int reps,
                                        float* ms_per_pass) {
    if (!h || !bgr_device || !ms_per_pass || n_frames < 1 || n_frames > h->max_batch || reps < 1 || width < 16 || height < 16 || width > h->max_w || height > h->max_h)
        return FID_ERR_INVALID_ARG;
    if (row_stride < (size_t)width * h->bpp || frame_stride < row_stride * (size_t)height || h->pend_count) return FID_ERR_INVALID_ARG;
    CK(cudaSetDevice(h->device));
    CK(cudaDeviceSynchronize());
    Slot& s = h->slot[0];
    const FrameGeom g = make_geom(h, width, height, row_stride, frame_stride);
    if (!h->t0) {
        CK(cudaEventCreate(&h->t0));
        CK(cudaEventCreate(&h->t1));
    }
    float total = 0.f;
    for (int r = -1; r < reps; r++) {  // one untimed pass first
        const int rc = enqueue_pipeline(h, s, h->stream, n_frames, g, bgr_device, nullptr, 0.0, 0, ST_THRESH);
        if (rc != FID_OK) return rc;
        CK(cudaStreamSynchronize(h->stream));
        float ms = 0.f;
        CK(cudaEventElapsedTime(&ms, s.ev[ST_THRESH], s.ev[ST_MASKS]));
        if (r >= 0) total += ms;
    }
    *ms_per_pass = total / (float)reps;
    return FID_OK;
}

extern "C" int fid_debug_candidates(fid_detector* h, int max_candidates, int* n, int32_t* quads, int32_t* scale, int32_t* contour_len) {
    if (!h || !n || h->pend_count) return FID_ERR_INVALID_ARG;
    CK(cudaSetDevice(h->device));
    Slot& s = h->slot[0];
    unsigned int cnt = 0;
    CK(cudaMemcpy(&cnt, s.d_nraw, sizeof(cnt), cudaMemcpyDeviceToHost));
    cnt = std::min<unsigned int>(cnt, (unsigned int)h->max_raw);
    std::vector<RawQuad> raw(cnt);
    if (cnt) CK(cudaMemcpy(raw.data(), s.d_raw, sizeof(RawQuad) * cnt, cudaMemcpyDeviceToHost));
    std::sort(raw.begin(), raw.end(), [](const RawQuad& a, const RawQuad& b) { return a.order_hi != b.order_hi ? a.order_hi < b.order_hi : a.order_lo < b.order_lo; });
    *n = (int)cnt;
    if ((int)cnt > max_candidates) return FID_ERR_CAPACITY;
    for (unsigned int i = 0; i < cnt; i++) {
        for (int k = 0; k < 4; k++) {
            if (quads) {
                quads[i * 8 + 2 * k] = raw[i].x[k];
                quads[i * 8 + 2 * k + 1] = raw[i].y[k];
            }
        }
        if (scale) scale[i] = (int)raw[i].order_hi;
        if (contour_len) contour_len[i] = raw[i].n_contour;
    }
    return FID_OK;
}

extern "C" int fid_last_stage_ms(fid_detector* h, float* ms, int max_stages, int* n_stages) {
    if (!h || !ms) return FID_ERR_INVALID_ARG;
    const int n = std::min(max_stages, (int)ST_COUNT + N_WALK_ROUNDS);
    for (int i = 0; i < n; i++) ms[i] = h->stage_ms[i];
    if (n_stages) *n_stages = ST_COUNT + N_WALK_ROUNDS;
    return FID_OK;
}

extern "C" int fid_last_counters(fid_detector* h, int64_t* counters, int max_counters, int* n_counters) {
    if (!h || !counters) return FID_ERR_INVALID_ARG;
    const int n = std::min(max_counters, 7);
    for (int i = 0; i < n; i++) counters[i] = h->counters[i];
    if (n_counters) *n_counters = 7;
    return FID_OK;
}
