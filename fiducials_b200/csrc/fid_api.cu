// C-ABI of the detector (include/fiducials_b200.h): handle management, batch orchestration on CUDA
// streams, stage timing.  No CPU fallback: every entry point that computes needs a CUDA device.
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <vector>

#include "../../include/fiducials_b200.h"
#include "kernels_contour.cuh"
#include "kernels_threshold.cuh"
#include "start_prune_table.h"
#include "kernels_threshold_mma.cuh"
#include "kernels_marker.cuh"
#include "kernels_aruco3.cuh"
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
    struct fid_pose_hypotheses* d_out_hyp = nullptr;  // fid_set_pose_hypotheses: allocated by the first enable
    fid_board_pose* d_out_board = nullptr;             // fid_set_boards: [max_batch][FID_MAX_BOARDS], allocated by the first set
    fid_charuco_result* d_out_ch = nullptr;            // fid_set_charuco_boards: [max_batch][FID_MAX_CHARUCO_BOARDS]
    int32_t* d_out_ch_ids = nullptr;                   // [max_batch][ch_slot_cap]
    float* d_out_ch_xy = nullptr;                      // [max_batch][ch_slot_cap][2]
    // fid_set_batch_marker_refinement: allocated by the first enable
    int32_t* d_rej_n = nullptr;                        // [max_batch]                 k_rejected
    float* d_rej = nullptr;                            // [max_batch][max_sel][8]
    int32_t* d_mr_nrec = nullptr;                      // [max_batch]                 k_marker_refine
    int32_t* d_mr_idx = nullptr;                       // [max_batch][max_markers]
    int32_t* d_mr_board = nullptr;                     // [max_batch][max_markers]
    int32_t* d_dia_n = nullptr;                        // fid_set_diamonds: [max_batch], allocated by the first enable
    fid_diamond* d_dia = nullptr;                      // [max_batch][FID_MAX_DIAMONDS]
    // fid_set_dictionaries: allocated when the handle enters multi-dictionary mode
    int32_t* d_md_count = nullptr;                     // [n_dicts][max_batch]             k_finish per dictionary
    int32_t* d_md_ids = nullptr;                       // [n_dicts][max_batch][max_markers]
    float* d_md_corners = nullptr;                     // [n_dicts][max_batch][max_markers][8]
    int32_t* d_out_dict = nullptr;                     // [max_batch][max_markers]          k_dict_merge
    int32_t* d_md_run = nullptr;                       // [max_batch][FID_MAX_DICTIONARIES + 1] k_dict_merge: each dictionary's run
    // fid_set_aruco3: allocated by the first enable (level 0 of the pyramid is d_gray)
    uint8_t* d_a3_pyr = nullptr;                       // [max_batch][levels 1.. of the largest frame]
    uint8_t* d_a3_seg = nullptr;                       // [max_batch][the largest segmentation plane of the mode's parameters]
    size_t a3_pyr_cap = 0, a3_seg_cap = 0;             // their sizes in bytes; fid_set_aruco3 grows them
    // detectMarkersWithConfidence (fid_set_marker_confidence / fid_detect_with_confidence): allocated by the first use
    float* d_cand_conf = nullptr;                      // [max_batch][max_sel]     k_identify_*<PYR, true>
    float* d_out_conf = nullptr;                       // [max_batch][max_markers] k_finish
    float* h_out_conf = nullptr;
    // pinned host mirrors
    int32_t* h_out_count = nullptr;
    int32_t* h_out_ids = nullptr;
    float* h_out_corners = nullptr;
    fid_transform* h_out_tf = nullptr;
    struct fid_pose_hypotheses* h_out_hyp = nullptr;
    fid_board_pose* h_out_board = nullptr;
    fid_charuco_result* h_out_ch = nullptr;
    int32_t* h_out_ch_ids = nullptr;
    float* h_out_ch_xy = nullptr;
    int ch_slot_cap = 0;
    int32_t* h_rej_n = nullptr;
    float* h_rej = nullptr;
    int32_t* h_mr_nrec = nullptr;
    int32_t* h_mr_idx = nullptr;
    int32_t* h_mr_board = nullptr;
    int32_t* h_dia_n = nullptr;
    fid_diamond* h_dia = nullptr;
    int32_t* h_out_dict = nullptr;
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
    // FID_STAGGER bit mask, see enqueue_pipeline.  Default 1: the threshold stages of consecutive chunks run one after the other
    // (C2 on H100: +2 % device-resident throughput, DESIGN.md section 5)
    int stagger = 1;
    int enc = FID_ENC_BGR8, bpp = 3;  // fid_set_input_encoding
    // fid_submit_batch / fid_collect_batch: FIFO of batches in flight
    struct Pending {
        int first_slot, n_chunks, n_frames, w, h;
        int64_t launches;
        bool pose, hyp, board, charuco, refine, diamonds, multi, conf;
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
    uint8_t* d_step_bytes = nullptr;  // bits 0-4 of both step tables, a byte per entry (k_walk / k_emit stage them into shared memory)
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
    // both planar pose hypotheses (fid_set_pose_hypotheses / fid_pose_hypotheses / fid_last_pose_hypotheses)
    int pose_hyp = 0;                                // the batch option
    struct fid_pose_hypotheses* d_hyp_list = nullptr;  // fid_pose_hypotheses output, 4096 records, allocated by the first call
    bool last_hyp_valid = false;                     // the batch last returned had the option on (and a camera)
    int last_hyp_frames = 0, last_hyp_stride = 0;
    std::vector<int32_t> last_hyp_counts;
    std::vector<struct fid_pose_hypotheses> last_hyp;  // [last_hyp_frames][last_hyp_stride]
    // one pose per board (fid_set_boards / fid_estimate_board_poses / fid_last_board_poses)
    int n_boards = 0;                                // 0 = off
    bool board_bound = false;                        // set with fid_set_family_boards: board_fam holds each board's dictionary index
    int32_t board_fam[FID_MAX_BOARDS]{};
    int32_t *d_board_off = nullptr, *d_board_keys = nullptr, *d_board_marker = nullptr;  // see BoardPoseArgs
    float* d_board_obj = nullptr;
    int32_t* d_board_count = nullptr;                // fid_estimate_board_poses: the list's length
    fid_board_pose* d_board_list = nullptr;          // fid_estimate_board_poses output, FID_MAX_BOARDS records
    bool last_board_valid = false;                   // the batch last returned had boards (and a camera)
    int last_board_frames = 0, last_board_n = 0;
    std::vector<fid_board_pose> last_board;          // [last_board_frames][last_board_n]
    // ChArUco boards (fid_set_charuco_boards / fid_detect_charuco / fid_last_charuco)
    int n_charuco = 0, charuco_slots = 0;            // 0 = off; slots = corners of all boards
    bool charuco_bound = false;                      // set with fid_set_family_charuco_boards
    int32_t charuco_fam[FID_MAX_CHARUCO_BOARDS]{};
    int32_t charuco_nm[FID_MAX_CHARUCO_BOARDS]{};    // each board's marker count (fid_set_dictionaries checks it against the family)
    CharucoBoardDev* d_ch_boards = nullptr;
    int32_t *d_ch_keys = nullptr, *d_ch_marker = nullptr, *d_ch_ids = nullptr, *d_ch_near_n = nullptr, *d_ch_near_idx = nullptr, *d_ch_near_corner = nullptr;
    float *d_ch_obj = nullptr, *d_ch_chess = nullptr, *d_ch_masks = nullptr;
    int32_t* d_ch_count = nullptr;                   // fid_detect_charuco: the list's length
    fid_charuco_result* d_ch_list = nullptr;         // fid_detect_charuco outputs
    int32_t* d_ch_list_ids = nullptr;
    float* d_ch_list_xy = nullptr;
    bool last_ch_valid = false;
    int last_ch_frames = 0, last_ch_n = 0, last_ch_slots = 0;
    std::vector<fid_charuco_result> last_ch;         // [last_ch_frames][last_ch_n]
    std::vector<int32_t> last_ch_ids;                // [last_ch_frames][last_ch_slots]
    std::vector<float> last_ch_xy;
    // recovery of missed board markers (fid_set_marker_refinement / fid_refine_detected_markers)
    fid_marker_refine_params mrefine{};              // enable = 0: off
    int32_t* d_mr_i = nullptr;                       // count, n_rejected, n_recovered, overflow, ids, recovered idx, recovered board
    float* d_mr_f = nullptr;                         // corners [FID_MAX_MARKERS][8], rejected [FID_MAX_REJECTED][8]
    int batch_refine = 0;                            // fid_set_batch_marker_refinement
    bool last_mr_valid = false;                      // the batch last returned refined (fid_last_marker_refinement)
    int last_mr_frames = 0;
    std::vector<int32_t> last_mr_nrec, last_mr_nrej;  // [last_mr_frames]
    std::vector<int32_t> last_mr_idx, last_mr_board;  // frame after frame, last_mr_nrec[f] each
    std::vector<float> last_mr_rej;                   // frame after frame, last_mr_nrej[f] x 8 each
    // ChArUco diamonds (fid_set_diamonds / fid_detect_diamonds / fid_last_diamonds)
    fid_diamond_params diamond{};                    // enable = 0: off
    bool diamond_bound = false;                      // set with fid_set_family_diamonds
    int32_t diamond_fam = 0;
    DiamondLayout diamond_layout{};
    int32_t* d_dia_io = nullptr;                     // fid_detect_diamonds: the list's length, the diamonds found
    fid_diamond* d_dia_list = nullptr;               // fid_detect_diamonds output, FID_MAX_DIAMONDS records
    bool last_dia_valid = false;                     // the batch last returned had diamonds (fid_last_diamonds)
    int last_dia_frames = 0;
    std::vector<int32_t> last_dia_n;                 // [last_dia_frames]
    std::vector<fid_diamond> last_dia;               // frame after frame, last_dia_n[f] each
    // several dictionaries (fid_set_dictionaries / fid_detect_multi_dict / fid_last_dict_indices)
    int n_dicts = 1;
    fid_dictionary_spec dict_spec[FID_MAX_DICTIONARIES]{};  // entry 0's dictionary is params.dictionary
    DevParams dict_P[FID_MAX_DICTIONARIES]{};        // params with each entry's dictionary
    bool multi = false;                              // more than one entry, or entry 0 with an offset or a length
    unsigned long long* d_mdict = nullptr;           // [FID_MAX_DICTIONARIES][kMaxDictMarkers * 4], multi-dictionary mode only
    bool last_di_valid = false;                      // fid_last_dict_indices
    int last_di_frames = 0, last_di_stride = 0;
    std::vector<int32_t> last_di_counts, last_di;    // [last_di_frames][last_di_stride]
    fid_aruco3_params aruco3{};                      // useAruco3Detection (fid_set_aruco3); enable = 0: off
    // detectMarkersWithConfidence (fid_set_marker_confidence / fid_detect_with_confidence / fid_last_marker_confidence)
    int marker_conf = 0;                             // the batch option
    bool last_conf_valid = false;                    // the batch last returned had the option on
    int last_conf_frames = 0, last_conf_stride = 0;
    std::vector<int32_t> last_conf_counts;
    std::vector<float> last_conf;                    // [last_conf_frames][last_conf_stride]
    bool detected_multi = false;                     // slot 0 holds fid_detect_multi_dict's candidates, not detectMarkers'
    int inverted = 0;                                // detectInvertedMarker (fid_set_detect_inverted_marker)
    int32_t* d_dbg_rej_n = nullptr;                  // fid_debug_rejected: count, then [max_sel][8] floats
    float* d_dbg_rej = nullptr;
    float stage_ms[ST_COUNT + N_WALK_ROUNDS]{};
    int64_t counters[8]{};
    cudaEvent_t t0 = nullptr, t1 = nullptr;
    // last geometry (for debug calls)
    int last_w = 0, last_h = 0, last_frames = 0;
    bool detected = false;  // fid_detect has run: slot 0 holds a frame's candidates (fid_debug_rejected)
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
    for (auto k : {k_sort_group<false>, k_sort_group<true>}) CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)group_smem(FID_GROUP_MAX_RAW)));
    for (auto k : {k_identify_retry<false>, k_identify_retry<true>, k_identify_retry<false, true>, k_identify_retry<true, true>, k_identify_retry<false, false, true>,
                   k_identify_retry<true, false, true>, k_identify_retry<false, true, true>, k_identify_retry<true, true, true>})
        CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kMaxDictMarkers * 4 * 8 + IDENT_WARPS * 256 * 4 + IDENT_WARPS * FID_MAX_WARP_SIDE_SQ)));
    for (auto k : {k_identify_first<false>, k_identify_first<true>, k_identify_first<false, true>, k_identify_first<true, true>, k_identify_first<false, false, true>,
                   k_identify_first<true, false, true>, k_identify_first<false, true, true>, k_identify_first<true, true, true>})
        CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kMaxDictMarkers * 4 * 8 + IDENT0_WARPS * 256 * 4 + IDENT0_WARPS * FID_MAX_WARP_SIDE_SQ)));
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
                     s.d_out_tf,      s.fs.raw_of_sorted, s.d_cand_raw,     s.d_first_list,   s.d_retry_list, s.d_out_hyp, s.d_out_board, s.d_out_ch, s.d_out_ch_ids, s.d_out_ch_xy,
                     s.d_rej_n,       s.d_rej,           s.d_mr_nrec,       s.d_mr_idx,       s.d_mr_board,    s.d_dia_n,       s.d_dia,
                     s.d_md_count,    s.d_md_ids,        s.d_md_corners,    s.d_out_dict,     s.d_md_run,      s.d_a3_pyr,      s.d_a3_seg,      s.d_cand_conf,   s.d_out_conf};
    for (void* p : dptrs)
        if (p) cudaFree(p);
    void* hptrs[] = {s.h_out_count, s.h_out_ids, s.h_out_corners, s.h_out_tf, s.h_counters, s.h_nsel, s.h_nrawc, s.h_out_hyp, s.h_out_board, s.h_out_ch, s.h_out_ch_ids, s.h_out_ch_xy,
                     s.h_rej_n,     s.h_rej,     s.h_mr_nrec,    s.h_mr_idx,   s.h_mr_board, s.h_dia_n, s.h_dia, s.h_out_dict, s.h_out_conf};
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
    h->dict_spec[0].dictionary = params->dictionary;
    h->dict_P[0] = P;
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
    // Start cracks: at most one left and one right crack per two pixels of a row and plane (halo_row_starts), i.e.
    // n_scales / 2 per pixel and side -- 6.5 with the reference's 13 scales.  Uniform noise gives 1.6, marker scenes 0.15;
    // a 1-pixel checkerboard or dither reaches the bound.  The queue holds 3 per pixel and side: a chunk with more is
    // walked again from its stored planes in groups of scales that fit (k_rescan_starts), so its result does not change.
    // In-range contour points: 3.6 per pixel on uniform noise (marker scenes 0.4); past the capacity, FID_ERR_CAPACITY.
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
        std::vector<uint8_t> sb(2 * FID_LUT_SIZE);
        build_step_bytes(sb.data(), sb.data() + FID_LUT_SIZE);
        if ((rc = dalloc(&h->d_step_bytes, sb.size())) != FID_OK) {
            fid_destroy(h);
            return rc;
        }
        CKH(cudaMemcpy(h->d_step_bytes, sb.data(), sb.size(), cudaMemcpyHostToDevice));
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
    void* ptrs[] = {h->d_prune, h->d_dict, h->d_pf[0], h->d_pf[1], h->d_lut_prev, h->d_lut_next, h->d_step_bytes, h->d_subpix_masks, h->d_override_ids, h->d_override_lens, h->d_pose_ids, h->d_pose_corners, h->d_pose_out, h->d_hyp_list,
                     h->d_board_off, h->d_board_keys, h->d_board_marker, h->d_board_obj, h->d_board_count, h->d_board_list, h->d_ch_boards, h->d_ch_keys,
                     h->d_ch_marker, h->d_ch_ids, h->d_ch_near_n, h->d_ch_near_idx, h->d_ch_near_corner, h->d_ch_obj, h->d_ch_chess, h->d_ch_masks,
                     h->d_ch_count, h->d_ch_list, h->d_ch_list_ids, h->d_ch_list_xy, h->d_mr_i, h->d_mr_f, h->d_dbg_rej_n, h->d_dbg_rej, h->d_dia_io, h->d_dia_list, h->d_mdict};
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

// DevParams of the first n dictionary entries under params p: entry 0 takes p.dictionary, entry d > 0 specs[d].dictionary.
static int dict_params(const fid_params& p, int n, const fid_dictionary_spec* specs, DevParams* out) {
    for (int d = 0; d < n; d++) {
        fid_params q = p;
        if (d > 0) q.dictionary = specs[d].dictionary;
        const int rc = make_dev_params(q, &out[d]);
        if (rc != FID_OK) return rc;
    }
    return FID_OK;
}

// multi-dictionary mode: every entry's table -> device, entry d at d * kMaxDictMarkers * 4 words
static int upload_dictionaries(fid_detector* h) {
    std::vector<unsigned long long> words;
    for (int d = 0; d < h->n_dicts; d++) {
        pack_dictionary(h->dict_P[d], &words);
        CK(cudaMemcpy(h->d_mdict + (size_t)d * kMaxDictMarkers * 4, words.data(), words.size() * sizeof(unsigned long long), cudaMemcpyHostToDevice));
    }
    return FID_OK;
}

extern "C" int fid_set_params(fid_detector* h, const fid_params* params) {
    if (!h || !params) return FID_ERR_INVALID_ARG;
    DevParams P;
    int rc = make_dev_params(*params, &P);
    if (rc != FID_OK) return rc;
    if (h->pend_count) return FID_ERR_INVALID_ARG;  // between frames only (configCallback, aruco_detect.cpp:257-298)
    DevParams dp[FID_MAX_DICTIONARIES];             // entries 1.. keep their dictionaries under the new parameters (cv2's setDictionary)
    if (h->n_dicts > 1 && (rc = dict_params(*params, h->n_dicts, h->dict_spec, dp)) != FID_OK) return rc;
    if ((int64_t)h->dict_spec[0].id_offset + P.n_markers - 1 > INT32_MAX) return FID_ERR_INVALID_ARG;  // entry 0's published ids
    CK(cudaSetDevice(h->device));
    for (int i = 0; i < h->n_slots; i++) CK(cudaStreamSynchronize(h->slot_stream[i]));
    CK(cudaStreamSynchronize(h->stream));
    h->params = *params;
    h->P = P;
    h->dict_spec[0].dictionary = params->dictionary;
    h->dict_P[0] = P;
    for (int d = 1; d < h->n_dicts; d++) h->dict_P[d] = dp[d];
    if ((rc = upload_dictionary(h)) != FID_OK) return rc;
    return h->multi ? upload_dictionaries(h) : FID_OK;
}

extern "C" int fid_set_dictionaries(fid_detector* h, int n, const fid_dictionary_spec* specs) {
    if (!h || !specs || n < 1 || n > FID_MAX_DICTIONARIES || h->pend_count) return FID_ERR_INVALID_ARG;
    fid_params p = h->params;
    p.dictionary = specs[0].dictionary;
    DevParams dp[FID_MAX_DICTIONARIES];
    int rc = dict_params(p, n, specs, dp);
    if (rc != FID_OK) return rc;
    for (int d = 0; d < n; d++) {
        if (!std::isfinite(specs[d].fiducial_len) || specs[d].fiducial_len < 0) return FID_ERR_INVALID_ARG;
        if ((int64_t)specs[d].id_offset + dp[d].n_markers - 1 > INT32_MAX) return FID_ERR_INVALID_ARG;  // a published id would overflow
    }
    const bool multi = n > 1 || specs[0].id_offset != 0 || specs[0].fiducial_len > 0;
    // a board set without a family is ambiguous with several dictionaries
    if (multi && ((h->n_boards && !h->board_bound) || (h->n_charuco && !h->charuco_bound) || (h->diamond.enable && !h->diamond_bound) || h->batch_refine ||
                  h->aruco3.enable || h->marker_conf))
        return FID_ERR_UNSUPPORTED;
    // every bound family must still exist, and a ChArUco board must fit its family's dictionary
    for (int b = 0; b < h->n_boards; b++)
        if (h->board_bound && h->board_fam[b] >= n) return FID_ERR_INVALID_ARG;
    for (int b = 0; b < h->n_charuco; b++)
        if (h->charuco_bound && (h->charuco_fam[b] >= n || h->charuco_nm[b] > dp[h->charuco_fam[b]].n_markers)) return FID_ERR_INVALID_ARG;
    if (h->diamond.enable && h->diamond_bound && h->diamond_fam >= n) return FID_ERR_INVALID_ARG;
    CK(cudaSetDevice(h->device));
    if (multi) {  // (a failed allocation leaves the handle as it was; the next call completes it)
        const size_t F = h->max_batch, M = F * h->max_markers, ND = FID_MAX_DICTIONARIES;
        if (!h->d_mdict && (rc = dalloc(&h->d_mdict, ND * kMaxDictMarkers * 4)) != FID_OK) return rc;
        for (int i = 0; i < h->n_slots; i++) {
            Slot& s = h->slot[i];
            if (!s.d_md_count && (rc = dalloc(&s.d_md_count, ND * F)) != FID_OK) return rc;
            if (!s.d_md_ids && (rc = dalloc(&s.d_md_ids, ND * M)) != FID_OK) return rc;
            if (!s.d_md_corners && (rc = dalloc(&s.d_md_corners, ND * M * 8)) != FID_OK) return rc;
            if (!s.d_out_dict && (rc = dalloc(&s.d_out_dict, M)) != FID_OK) return rc;
            if (!s.d_md_run && (rc = dalloc(&s.d_md_run, F * (ND + 1))) != FID_OK) return rc;
            if (!s.h_out_dict && (rc = halloc(&s.h_out_dict, M)) != FID_OK) return rc;
        }
    }
    for (int i = 0; i < h->n_slots; i++) CK(cudaStreamSynchronize(h->slot_stream[i]));
    CK(cudaStreamSynchronize(h->stream));
    h->params = p;
    h->P = dp[0];
    h->n_dicts = n;
    h->multi = multi;
    for (int d = 0; d < n; d++) {
        h->dict_spec[d] = specs[d];
        h->dict_P[d] = dp[d];
    }
    if ((rc = upload_dictionary(h)) != FID_OK) return rc;
    return multi ? upload_dictionaries(h) : FID_OK;
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
static BoardPoseArgs board_args(const fid_detector* h, const int32_t* count, const int32_t* ids, const float* corners, int max_markers, const fid_camera* cam,
                                fid_board_pose* out) {
    BoardPoseArgs a{};
    a.max_markers = max_markers;
    a.n_boards = h->n_boards;
    a.count = count;
    a.ids = ids;
    a.corners = corners;
    a.board_off = h->d_board_off;
    a.board_keys = h->d_board_keys;
    a.board_marker = h->d_board_marker;
    a.board_obj = h->d_board_obj;
    for (int b = 0; b < h->n_boards; b++) a.family[b] = h->board_fam[b];
    a.cam = make_camera(cam);
    a.out = out;
    return a;
}

static CharucoArgs charuco_args(const fid_detector* h, const uint8_t* src, size_t row_stride, size_t frame_stride, int W, int H, const int32_t* count, const int32_t* ids,
                                const float* corners, int max_markers, const fid_camera* cam, fid_charuco_result* out, int32_t* out_ids, float* out_xy) {
    CharucoArgs a{};
    a.src = src;
    a.row_stride = row_stride;
    a.frame_stride = frame_stride;
    a.enc = h->enc;
    a.W = W;
    a.H = H;
    a.max_markers = max_markers;
    a.count = count;
    a.ids = ids;
    a.corners = corners;
    a.n_boards = h->n_charuco;
    a.n_slots = h->charuco_slots;
    a.boards = h->d_ch_boards;
    a.keys = h->d_ch_keys;
    a.marker_of = h->d_ch_marker;
    a.board_ids = h->d_ch_ids;
    a.obj = h->d_ch_obj;
    a.chess = h->d_ch_chess;
    a.near_n = h->d_ch_near_n;
    a.near_idx = h->d_ch_near_idx;
    a.near_corner = h->d_ch_near_corner;
    a.masks = h->d_ch_masks;
    // cornerSubPix's own clamps of the criteria (MIN(MAX(maxCount, 1), 100), MAX(epsilon, 0)^2); the detector's window is used
    // where no nearest marker is detected, within the 1..10 the mask table covers
    a.win_default = std::max(1, std::min(FID_CHARUCO_MAX_WIN, h->params.cornerRefinementWinSize));
    a.max_iters = std::max(1, std::min(100, h->params.cornerRefinementMaxIterations));
    const double eps = std::max(h->params.cornerRefinementMinAccuracy, 0.0);
    a.eps_sq = eps * eps;
    a.has_cam = cam ? 1 : 0;
    a.cam = make_camera(cam);
    a.out = out;
    a.out_ids = out_ids;
    a.out_xy = out_xy;
    return a;
}

// k_marker_refine's frames, parameters and boards; the caller sets the lists.
static MarkerRefineArgs marker_refine_args(const fid_detector* h, const uint8_t* src, size_t row_stride, size_t frame_stride, int W, int H, const fid_camera* cam) {
    MarkerRefineArgs a{};
    a.src = src;
    a.row_stride = row_stride;
    a.frame_stride = frame_stride;
    a.enc = h->enc;
    a.W = W;
    a.H = H;
    a.P = h->P;
    a.dict = h->d_dict;
    a.subpix_masks = h->d_subpix_masks;
    a.rp = MarkerRefineParams{h->mrefine.min_rep_distance, h->mrefine.error_correction_rate, h->mrefine.check_all_orders ? 1 : 0};
    a.n_boards = h->n_boards;
    a.board_off = h->d_board_off;
    a.board_keys = h->d_board_keys;
    a.board_marker = h->d_board_marker;
    a.board_obj = h->d_board_obj;
    a.n_charuco = h->n_charuco;
    a.ch_boards = h->d_ch_boards;
    a.ch_keys = h->d_ch_keys;
    a.ch_marker = h->d_ch_marker;
    a.ch_obj = h->d_ch_obj;
    a.has_cam = cam ? 1 : 0;
    a.cam = make_camera(cam);
    return a;
}

// k_diamond's frames and parameters; the caller sets the lists.
static DiamondArgs diamond_args(const fid_detector* h, const uint8_t* src, size_t row_stride, size_t frame_stride, int W, int H, const fid_camera* cam) {
    DiamondArgs a{};
    a.src = src;
    a.row_stride = row_stride;
    a.frame_stride = frame_stride;
    a.enc = h->enc;
    a.W = W;
    a.H = H;
    a.P = h->dict_P[h->diamond_fam];  // the cornerSubPix of the markers the loop takes reads the family's parameters
    a.family = h->diamond_fam;
    a.id_offset = h->dict_spec[h->diamond_fam].id_offset;
    a.subpix_masks = h->d_subpix_masks;
    a.ch_masks = h->d_ch_masks;
    a.layout = h->diamond_layout;
    a.win_default = std::max(1, std::min(FID_CHARUCO_MAX_WIN, h->params.cornerRefinementWinSize));  // as charuco_args
    a.max_iters = std::max(1, std::min(100, h->params.cornerRefinementMaxIterations));
    const double eps = std::max(h->params.cornerRefinementMinAccuracy, 0.0);
    a.eps_sq = eps * eps;
    a.has_cam = cam ? 1 : 0;
    a.cam = make_camera(cam);
    return a;
}

// A batch refines only with the batch switch, the refinement parameters and a board to refine against.
static bool batch_refines(const fid_detector* h) { return h->batch_refine && h->mrefine.enable && h->n_boards + h->n_charuco > 0; }

// useAruco3Detection (fid_set_aruco3): the gray plane (k_gray into d_gray, level 0), the pyrDown levels and the segmentation plane
// of nf frames.  Returns the number of launches.
static int enqueue_aruco3_planes(const fid_detector* h, Slot& s, cudaStream_t st, int nf, const FrameGeom& g, const uint8_t* d_bgr, const A3Geom& ag) {
    GrayArgs ga{};
    ga.bgr = d_bgr;
    ga.gray = s.d_gray;
    ga.W = g.W;
    ga.H = g.H;
    ga.n_frames = nf;
    ga.bgr_row_stride = g.bgr_row_stride;
    ga.bgr_frame_stride = g.bgr_frame_stride;
    ga.gray_pitch = g.gray_pitch;
    ga.gray_frame_stride = g.gray_frame_stride;
    ga.enc = h->enc;
    const long long gq = (long long)nf * g.H * ((g.W + 3) / 4);
    k_gray<<<(unsigned int)((gq + 255) / 256), 256, 0, st>>>(ga);
    int launches = 1;
    for (int l = 1; l < ag.n_levels; l++) {
        A3PlaneArgs a{};
        a.src = l == 1 ? s.d_gray : s.d_a3_pyr + ag.lv[l - 1].off;
        a.src_pitch = ag.lv[l - 1].pitch;
        a.src_frame_stride = l == 1 ? g.gray_frame_stride : ag.pyr_frame_bytes;
        a.sw = ag.lv[l - 1].W;
        a.sh = ag.lv[l - 1].H;
        a.dst = s.d_a3_pyr + ag.lv[l].off;
        a.dst_pitch = ag.lv[l].pitch;
        a.dst_frame_stride = ag.pyr_frame_bytes;
        a.dw = ag.lv[l].W;
        a.dh = ag.lv[l].H;
        a.n_frames = nf;
        k_a3_pyr_down<<<dim3((a.dw + 255) / 256, a.dh, nf), 256, 0, st>>>(a);
        launches++;
    }
    if (ag.resized) {
        A3PlaneArgs a{};
        a.src = s.d_gray;
        a.src_pitch = g.gray_pitch;
        a.src_frame_stride = g.gray_frame_stride;
        a.sw = g.W;
        a.sh = g.H;
        a.dst = s.d_a3_seg;
        a.dst_pitch = ag.seg_w;
        a.dst_frame_stride = (size_t)ag.seg_w * ag.seg_h;
        a.dw = ag.seg_w;
        a.dh = ag.seg_h;
        a.n_frames = nf;
        a.scale_x = 1.0 / ((double)ag.seg_w / g.W);
        a.scale_y = 1.0 / ((double)ag.seg_h / g.H);
        k_a3_resize<<<dim3((a.dw + 255) / 256, a.dh, nf), 256, 0, st>>>(a);
        launches++;
    }
    return launches;
}

static int enqueue_pipeline(fid_detector* h, Slot& s, cudaStream_t st, int nf, const FrameGeom& g, const uint8_t* d_bgr, const fid_camera* cam, double fiducial_len,
                            int n_override, int stop_after /* -1 = all */, const Slot* prev = nullptr, bool refine = false, bool diamonds = false,
                            bool multi = false, bool conf = false) {
    const DevParams& P = h->P;
    int launches = 0;
    CK(cudaMemsetAsync(s.d_counters, 0, sizeof(Counters), st));
    CK(cudaMemsetAsync(s.d_nraw, 0, sizeof(unsigned int) * nf, st));
    // stagger: a stage of this chunk starts after the same stage of the previous chunk has finished, so the
    // low-occupancy tails of one chunk (last walk round, grouping, identification, pose) run under the
    // throughput-bound stages of the other instead of under its own twin
    if (prev && (h->stagger & 1)) CK(cudaStreamWaitEvent(st, prev->ev[ST_MASKS], 0));
    CK(cudaEventRecord(s.ev[ST_THRESH], st));
    // useAruco3Detection: the stages up to k_finish run on the segmentation plane, a mono8 frame of its own size (gs, seg_src).
    // The threshold-only runs (fid_debug_threshold, fid_debug_time_threshold) stay on the full frame.
    const bool a3 = h->aruco3.enable != 0 && stop_after != ST_THRESH;
    const bool inv = h->inverted != 0;  // detectInvertedMarker: grouping and identification run their INV instantiations
    A3Geom ag{};
    FrameGeom gs = g;
    const uint8_t* seg_src = d_bgr;
    int seg_enc = h->enc;
    if (a3) {
        if (!a3_geometry(g.W, g.H, h->aruco3.minSideLengthCanonicalImg, h->aruco3.minMarkerLengthRatioOriginalImg, &ag)) return FID_ERR_INVALID_ARG;
        if ((size_t)nf * ag.pyr_frame_bytes > s.a3_pyr_cap || (ag.resized && (size_t)nf * ag.seg_w * ag.seg_h > s.a3_seg_cap)) return FID_ERR_CAPACITY;  // see a3_plane_bytes
        launches += enqueue_aruco3_planes(h, s, st, nf, g, d_bgr, ag);
        seg_src = ag.resized ? s.d_a3_seg : s.d_gray;
        const size_t pitch = ag.resized ? (size_t)ag.seg_w : (size_t)g.gray_pitch;
        gs = make_geom(h, ag.seg_w, ag.seg_h, pitch, pitch * ag.seg_h);
        seg_enc = FID_ENC_MONO8;
    }
    const int W = gs.W, H = gs.H;
    bool padded_starts = false;  // the tensor-core kernel queues start cracks in blocks padded with null records
    {  // threshold stage: gray + 13 adaptive thresholds -> halo tiles + start cracks
        bool fast = P.n_scales == 13;
        for (int i = 0; i < P.n_scales; i++) fast = fast && P.win[i] == 3 + 4 * i;
        if (fast && h->thresh_mode == 1) {
            // tensor-core kernel: persistent, one CTA per SM; BGR staged by TMA where the layout allows
            ThreshMmaArgs a{};
            a.src = seg_src;
            a.enc = seg_enc;
            a.bpp = seg_enc == FID_ENC_MONO8 ? 1 : 3;
            a.row_stride = gs.bgr_row_stride;
            a.frame_stride = gs.bgr_frame_stride;
            a.halo = s.d_halo;
            a.W = W;
            a.H = H;
            a.n_frames = nf;
            a.halo_tpr = gs.halo_tpr;
            a.halo_tiles_y = gs.halo_tiles_y;
            a.halo_scale_stride = gs.halo_scale_stride;
            a.halo_frame_stride = gs.halo_frame_stride;
            a.thresh_c = P.thresh_c;
            a.tiles_x = (gs.halo_tpr + THR_TILES_X - 1) / THR_TILES_X;
            a.tiles_y = (gs.halo_tiles_y + THR_TILES_Y - 1) / THR_TILES_Y;
            a.starts = s.d_starts;
            a.counters = s.d_counters;
            a.max_starts = h->max_starts;
            CUtensorMap tmap;
            memset(&tmap, 0, sizeof(tmap));
            static const bool tma_off = getenv("FID_THRESH_TMA") && atoi(getenv("FID_THRESH_TMA")) == 0;  // debugging switch
            padded_starts = true;
            a.use_tma = (!tma_off && seg_enc != FID_ENC_MONO8 && make_bgr_tensor_map(&tmap, seg_src, W, H, nf, gs.bgr_row_stride, gs.bgr_frame_stride)) ? 1 : 0;
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
            a.src = seg_src;
            a.src_row_stride = gs.bgr_row_stride;
            a.src_frame_stride = gs.bgr_frame_stride;
            a.enc = seg_enc;
            a.aligned4 = (W % 4 == 0) && (gs.bgr_row_stride % 4 == 0) && (gs.bgr_frame_stride % 4 == 0) && ((uintptr_t)seg_src % 4 == 0);
            a.halo = s.d_halo;
            a.W = W;
            a.H = H;
            a.n_frames = nf;
            a.halo_tpr = gs.halo_tpr;
            a.halo_tiles_y = gs.halo_tiles_y;
            a.halo_scale_stride = gs.halo_scale_stride;
            a.halo_frame_stride = gs.halo_frame_stride;
            a.n_scales = P.n_scales;
            a.r_max = r_max_of(P);
            a.thresh_c = P.thresh_c;
            a.starts = s.d_starts;
            a.counters = s.d_counters;
            a.max_starts = h->max_starts;
            a.prune = h->start_prune ? h->d_prune : nullptr;
            for (int i = 0; i < P.n_scales; i++) a.win[i] = P.win[i];
            dim3 grid((gs.halo_tpr + THR_TILES_X - 1) / THR_TILES_X, (gs.halo_tiles_y + THR_TILES_Y - 1) / THR_TILES_Y, nf);
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
    // useAruco3Detection replaces minMarkerPerimeterRate by a minimum contour length of 4 * minSideLengthCanonicalImg
    const int min_len = a3 ? 4 * h->aruco3.minSideLengthCanonicalImg : (int)(P.min_perimeter_rate * mx), max_len = (int)(P.max_perimeter_rate * mx);
    {  // walk, in rounds of growing budget
        WalkArgs a{};
        a.halo = s.d_halo;
        a.lut_prev = h->d_lut_prev;
        a.lut_next = h->d_lut_next;
        a.step_bytes = h->d_step_bytes;
        a.starts = s.d_starts;
        a.chains = s.d_chains;
        a.segs = s.d_segs;
        a.max_segs = h->max_segs;
        a.counters = s.d_counters;
        a.max_starts = h->max_starts;
        a.max_chains = h->max_chains;
        a.max_points = h->max_points;
        a.max_queue = h->max_queue;
        a.g = gs;
        a.min_len = min_len;
        a.max_len = max_len;
        // the rounds over the start queue of the threshold kernel (replay_group -1) or of one scale group of the replay
        auto walk_rounds = [&](int replay_group, bool timed) {
            a.replay_group = replay_group;
            for (int r = 0; r < N_WALK_ROUNDS; r++) {
                if (timed) CK(cudaEventRecord(s.ev_round[r], st));
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
            return FID_OK;
        };
        if (int rc = walk_rounds(-1, true)) return rc;
        CK(cudaEventRecord(s.ev_round[N_WALK_ROUNDS], st));
        // start-queue replay (kernels_contour.cuh, k_rescan_starts): scale groups of at most `per_group` planes, so that a group's
        // start cracks -- at most ceil(W / 2) per row, plane and side -- fit the queue's max_starts / 2 per side.  Not enqueued
        // where the planes of one chunk cannot hold more cracks than that and the queue holds no padding.
        const size_t per_plane = (size_t)((W + 1) / 2) * H * nf, cap = h->max_starts / 2;
        if (padded_starts || per_plane * P.n_scales > cap) {
            const int per_group = (int)std::max<size_t>(1, std::min<size_t>(P.n_scales, cap / per_plane));
            RescanArgs ra{};
            ra.halo = s.d_halo;
            ra.starts = s.d_starts;
            ra.counters = s.d_counters;
            ra.max_starts = h->max_starts;
            ra.prune = h->start_prune ? h->d_prune : nullptr;
            ra.g = gs;
            ra.n_frames = nf;
            for (int g0 = 0, grp = 0; g0 < P.n_scales; g0 += per_group, grp++) {
                ra.s_lo = g0;
                ra.s_hi = std::min(P.n_scales, g0 + per_group);
                ra.group = grp;
                launch_prio(k_rescan_starts, dim3(h->sm_count * 8), dim3(256), 0, st, 1, ra);
                launches++;
                if (int rc = walk_rounds(grp, false)) return rc;
            }
        }
    }
    CK(cudaEventRecord(s.ev[ST_EMIT], st));
    {  // emit
        EmitArgs a{};
        a.halo = s.d_halo;
        a.step_bytes = h->d_step_bytes;
        a.segs = s.d_segs;
        a.points = s.d_points;
        a.counters = s.d_counters;
        a.work_counter = &s.d_counters->emit_work;
        a.max_segs = h->max_segs;
        a.g = gs;
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
    // grouping, identification, CORNER_REFINE_CONTOUR and k_finish for one dictionary's parameters and table
    auto group = [&](int marker_size) {
        GroupArgs a{};
        a.raw = s.d_raw;
        a.n_raw = s.d_nraw;
        a.fs = s.fs;
        a.n_sel = s.d_nsel;
        a.n_raw_clamped = s.d_nrawc;
        a.max_raw = h->max_raw;
        a.close_wpr = h->close_wpr;
        a.max_sel = h->max_sel;
        a.marker_size = marker_size;
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
        launch_prio(inv ? k_sort_group<true> : k_sort_group<false>, dim3(nf), dim3(GROUP_THREADS), group_smem(h->max_raw), st, 4, a);
        launches++;
    };
    auto identify = [&](const DevParams& Pd, const unsigned long long* dict) {
        IdentifyArgs a{};
        a.src = d_bgr;
        a.row_stride = g.bgr_row_stride;
        a.frame_stride = g.bgr_frame_stride;
        a.enc = h->enc;
        a.W = g.W;
        a.H = g.H;
        a.fs = s.fs;
        a.n_sel = s.d_nsel;
        a.max_raw = h->max_raw;
        a.max_sel = h->max_sel;
        a.P = Pd;
        a.dict = dict;
        a.cand_id = s.d_cand_id;
        a.cand_corners = s.d_cand_corners;
        a.cand_raw = s.d_cand_raw;
        a.first_list = s.d_first_list;
        a.retry_list = s.d_retry_list;
        a.counters = s.d_counters;
        // fixed grids over work lists: a grid of one block per (frame, candidate slot) is 32 768 blocks of which 1 500 have work
        if (a3) a.pyr = A3Pyramid{s.d_gray, g.gray_frame_stride, s.d_a3_pyr, s.d_raw, ag};
        if (inv) {  // detectInvertedMarker: [useAruco3Detection][detectMarkersWithConfidence]
            static void (*const first[2][2])(const IdentifyArgs) = {{k_identify_first<false, false, true>, k_identify_first<false, true, true>},
                                                                    {k_identify_first<true, false, true>, k_identify_first<true, true, true>}};
            static void (*const retry[2][2])(const IdentifyArgs) = {{k_identify_retry<false, false, true>, k_identify_retry<false, true, true>},
                                                                    {k_identify_retry<true, false, true>, k_identify_retry<true, true, true>}};
            if (conf) a.cand_conf = s.d_cand_conf;
            launch_prio(first[a3][conf], dim3(h->sm_count * 4), dim3(IDENT0_WARPS * 32), ident_smem(Pd, IDENT0_WARPS), st, 4, a);
            launch_prio(retry[a3][conf], dim3(h->sm_count * 2), dim3(IDENT_WARPS * 32), ident_smem(Pd, IDENT_WARPS), st, 4, a);
        } else if (conf) {  // detectMarkersWithConfidence
            a.cand_conf = s.d_cand_conf;
            launch_prio(a3 ? k_identify_first<true, true> : k_identify_first<false, true>, dim3(h->sm_count * 4), dim3(IDENT0_WARPS * 32), ident_smem(Pd, IDENT0_WARPS), st, 4, a);
            launch_prio(a3 ? k_identify_retry<true, true> : k_identify_retry<false, true>, dim3(h->sm_count * 2), dim3(IDENT_WARPS * 32), ident_smem(Pd, IDENT_WARPS), st, 4, a);
        } else if (a3) {
            launch_prio(k_identify_first<true>, dim3(h->sm_count * 4), dim3(IDENT0_WARPS * 32), ident_smem(Pd, IDENT0_WARPS), st, 4, a);
            launch_prio(k_identify_retry<true>, dim3(h->sm_count * 2), dim3(IDENT_WARPS * 32), ident_smem(Pd, IDENT_WARPS), st, 4, a);
        } else {
            launch_prio(k_identify_first<false>, dim3(h->sm_count * 4), dim3(IDENT0_WARPS * 32), ident_smem(Pd, IDENT0_WARPS), st, 4, a);
            launch_prio(k_identify_retry<false>, dim3(h->sm_count * 2), dim3(IDENT_WARPS * 32), ident_smem(Pd, IDENT_WARPS), st, 4, a);
        }
        launches += 2;
    };
    auto contour_refine = [&]() {  // CORNER_REFINE_CONTOUR: rewrite the decoded candidates' corners before the output stage
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
    };
    auto finish = [&](const DevParams& Pd, const fid_camera* fcam, int32_t* out_count, int32_t* out_ids, float* out_corners) {
        FinishArgs a{};
        a.src = d_bgr;
        a.row_stride = g.bgr_row_stride;
        a.frame_stride = g.bgr_frame_stride;
        a.enc = h->enc;
        a.W = g.W;
        a.H = g.H;
        a.n_sel = s.d_nsel;
        a.cand_id = s.d_cand_id;
        a.cand_corners = s.d_cand_corners;
        a.fs = s.fs;
        a.max_raw = h->max_raw;
        a.max_sel = h->max_sel;
        a.max_markers = h->max_markers;
        a.P = Pd;
        a.subpix_masks = h->d_subpix_masks;
        a.do_pose = fcam ? 1 : 0;
        a.cam = make_camera(fcam);
        a.fiducial_len = fiducial_len;
        a.n_override = n_override;
        a.override_ids = h->d_override_ids;
        a.override_lens = h->d_override_lens;
        a.out_count = out_count;
        a.out_ids = out_ids;
        a.out_corners = out_corners;
        a.out_tf = s.d_out_tf;
        a.counters = s.d_counters;
        launch_prio(k_finish, dim3(nf), dim3(FINISH_THREADS), 0, st, 5, a);
        launches++;
        if (conf) {  // detectMarkersWithConfidence: the candidates' confidences in marker order
            ConfGatherArgs ca{};
            ca.n_sel = s.d_nsel;
            ca.cand_id = s.d_cand_id;
            ca.cand_conf = s.d_cand_conf;
            ca.fs = s.fs;
            ca.max_raw = h->max_raw;
            ca.max_sel = h->max_sel;
            ca.max_markers = h->max_markers;
            ca.out_conf = s.d_out_conf;
            launch_prio(k_conf_gather, dim3(nf), dim3(FINISH_THREADS), 0, st, 5, ca);
            launches++;
        }
    };
    // The opt-in board stages over the frame's final markers.  run = nullptr: every marker; in multi-dictionary mode k_dict_merge's
    // per-frame runs, so that each board, ChArUco board and the diamonds read their family's markers alone.
    auto board_stages = [&](const int32_t* run) {
        if (h->n_boards && cam) {  // one pose per (frame, board) (fid_set_boards / fid_set_family_boards)
            BoardPoseArgs a = board_args(h, s.d_out_count, s.d_out_ids, s.d_out_corners, h->max_markers, cam, s.d_out_board);
            a.run = run;
            launch_prio(k_board_pose, dim3(nf * h->n_boards), dim3(FID_BOARD_LANES), 0, st, 5, a);
            launches++;
        }
        if (h->n_charuco) {  // ChArUco corners (and pose with a camera) per (frame, board) (fid_set_charuco_boards / fid_set_family_charuco_boards)
            CharucoArgs a = charuco_args(h, d_bgr, g.bgr_row_stride, g.bgr_frame_stride, g.W, g.H, s.d_out_count, s.d_out_ids, s.d_out_corners, h->max_markers, cam,
                                         s.d_out_ch, s.d_out_ch_ids, s.d_out_ch_xy);
            a.run = run;
            launch_prio(k_charuco, dim3(nf * h->n_charuco), dim3(CHARUCO_THREADS), CHARUCO_SMEM, st, 5, a);
            launches++;
        }
        if (diamonds) {  // ChArUco diamonds per frame, from the final markers (fid_set_diamonds / fid_set_family_diamonds)
            DiamondArgs a = diamond_args(h, d_bgr, g.bgr_row_stride, g.bgr_frame_stride, g.W, g.H, cam);
            a.max_markers = h->max_markers;
            a.count = s.d_out_count;
            a.ids = s.d_out_ids;
            a.corners = s.d_out_corners;
            a.run = run;
            a.n_out = s.d_dia_n;
            a.out = s.d_dia;
            launch_prio(k_diamond, dim3(nf), dim3(DIAMOND_THREADS), 0, st, 5, a);
            launches++;
        }
    };
    if (multi) {  // several dictionaries (fid_set_dictionaries): the front end above ran once
        const size_t F = h->max_batch, dstride = F * h->max_markers;
        int grouped = -1;
        for (int d = 0; d < h->n_dicts; d++) {
            const DevParams& Pd = h->dict_P[d];
            if (Pd.marker_size != grouped) {  // filterTooCloseCandidates depends on the marker size only
                CK(cudaMemsetAsync(&s.d_counters->n_first, 0, sizeof(unsigned int), st));
                group(Pd.marker_size);
                grouped = Pd.marker_size;
            }
            CK(cudaMemsetAsync(&s.d_counters->n_retry, 0, sizeof(unsigned int), st));
            identify(Pd, h->d_mdict + (size_t)d * kMaxDictMarkers * 4);
            if (Pd.corner_refine == 2) contour_refine();
            finish(Pd, nullptr, s.d_md_count + d * F, s.d_md_ids + d * dstride, s.d_md_corners + d * dstride * 8);
        }
        // the stages interleave per dictionary: ST_GROUP holds all of them, ST_IDENT is empty, ST_SUBPIX_POSE is the merge
        CK(cudaEventRecord(s.ev[ST_IDENT], st));
        CK(cudaEventRecord(s.ev[ST_SUBPIX_POSE], st));
        DictMergeArgs a{};
        a.n_dicts = h->n_dicts;
        a.dict_stride = dstride;
        a.count = s.d_md_count;
        a.ids = s.d_md_ids;
        a.corners = s.d_md_corners;
        a.F = (int)F;
        a.max_markers = h->max_markers;
        for (int d = 0; d < h->n_dicts; d++) {
            a.dp[d].id_offset = h->dict_spec[d].id_offset;
            a.dp[d].len = h->dict_spec[d].fiducial_len > 0 ? h->dict_spec[d].fiducial_len : fiducial_len;
        }
        a.do_pose = cam ? 1 : 0;
        a.cam = make_camera(cam);
        a.n_override = n_override;
        a.override_ids = h->d_override_ids;
        a.override_lens = h->d_override_lens;
        a.out_count = s.d_out_count;
        a.out_ids = s.d_out_ids;
        a.out_corners = s.d_out_corners;
        a.out_dict = s.d_out_dict;
        a.out_run = s.d_md_run;
        a.out_tf = s.d_out_tf;
        a.out_hyp = (h->pose_hyp && cam) ? s.d_out_hyp : nullptr;
        a.counters = s.d_counters;
        launch_prio(k_dict_merge, dim3(nf), dim3(DICT_MERGE_THREADS), 0, st, 5, a);
        launches++;
        board_stages(s.d_md_run);
        CK(cudaEventRecord(s.ev[ST_D2H], st));
        h->counters[6] += launches;
        CK(cudaGetLastError());
        return FID_OK;
    }
    group(P.marker_size);
    CK(cudaEventRecord(s.ev[ST_IDENT], st));
    identify(P, h->d_dict);
    CK(cudaEventRecord(s.ev[ST_SUBPIX_POSE], st));
    if (a3) {  // k_finish without refinement or pose, then findCornerInPyrImage and the poses on the full-resolution corners
        DevParams Pf = P;
        Pf.corner_refine = 0;
        finish(Pf, nullptr, s.d_out_count, s.d_out_ids, s.d_out_corners);
        A3CornerArgs ca{};
        ca.pyr = A3Pyramid{s.d_gray, g.gray_frame_stride, s.d_a3_pyr, s.d_raw, ag};
        ca.count = s.d_out_count;
        ca.corners = s.d_out_corners;
        ca.max_markers = h->max_markers;
        ca.subpix_masks = h->d_subpix_masks;
        ca.max_iters = P.refine_max_iter;
        ca.eps_sq = P.refine_min_acc * P.refine_min_acc;
        launch_prio(k_a3_corners, dim3(nf), dim3(FINISH_THREADS), 0, st, 5, ca);
        launches++;
        if (cam) {
            RecoveredPoseArgs pa{};
            pa.count = s.d_out_count;
            pa.n_rec = s.d_out_count;  // every marker of the frame
            pa.ids = s.d_out_ids;
            pa.corners = s.d_out_corners;
            pa.max_markers = h->max_markers;
            pa.cam = make_camera(cam);
            pa.fiducial_len = fiducial_len;
            pa.n_override = n_override;
            pa.override_ids = h->d_override_ids;
            pa.override_lens = h->d_override_lens;
            pa.out_tf = s.d_out_tf;
            launch_prio(k_recovered_pose, dim3(nf), dim3(32), 0, st, 5, pa);
            launches++;
        }
    } else {
        if (P.corner_refine == 2) contour_refine();
        finish(P, cam, s.d_out_count, s.d_out_ids, s.d_out_corners);
    }
    if (refine) {  // opt-in: recover missed board markers before the stages that read the markers (fid_set_batch_marker_refinement)
        RejectedArgs ra{};
        ra.n_sel = s.d_nsel;
        ra.cand_id = s.d_cand_id;
        ra.fs = s.fs;
        ra.max_raw = h->max_raw;
        ra.max_sel = h->max_sel;
        ra.n_rej = s.d_rej_n;
        ra.rej = s.d_rej;
        launch_prio(k_rejected, dim3(nf), dim3(FINISH_THREADS), 0, st, 5, ra);
        MarkerRefineArgs a = marker_refine_args(h, d_bgr, g.bgr_row_stride, g.bgr_frame_stride, g.W, g.H, cam);
        a.n_rej = s.d_rej_n;
        a.rej = s.d_rej;
        a.max_rej = h->max_sel;
        a.max_markers = h->max_markers;
        a.count = s.d_out_count;
        a.ids = s.d_out_ids;
        a.corners = s.d_out_corners;
        a.n_rec = s.d_mr_nrec;
        a.rec_idx = s.d_mr_idx;
        a.rec_board = s.d_mr_board;
        a.overflow = &s.d_counters->overflow;
        launch_prio(k_marker_refine, dim3(nf), dim3(MREFINE_THREADS), MREFINE_SMEM, st, 5, a);
        launches += 2;
        if (cam) {
            RecoveredPoseArgs pa{};
            pa.count = s.d_out_count;
            pa.n_rec = s.d_mr_nrec;
            pa.ids = s.d_out_ids;
            pa.corners = s.d_out_corners;
            pa.max_markers = h->max_markers;
            pa.cam = make_camera(cam);
            pa.fiducial_len = fiducial_len;
            pa.n_override = n_override;
            pa.override_ids = h->d_override_ids;
            pa.override_lens = h->d_override_lens;
            pa.out_tf = s.d_out_tf;
            launch_prio(k_recovered_pose, dim3(nf), dim3(32), 0, st, 5, pa);
            launches++;
        }
    }
    if (h->pose_hyp && cam) {  // opt-in: both planar hypotheses of every marker k_finish wrote (fid_set_pose_hypotheses)
        PoseHypArgs a{};
        a.nf = nf;
        a.max_markers = h->max_markers;
        a.count = s.d_out_count;
        a.corners = s.d_out_corners;
        a.tf = s.d_out_tf;
        a.cam = make_camera(cam);
        a.fiducial_len = fiducial_len;
        a.n_override = n_override;
        a.override_ids = h->d_override_ids;
        a.override_lens = h->d_override_lens;
        a.out = s.d_out_hyp;
        launch_prio(k_pose_hypotheses, dim3(nf), dim3(POSE_HYP_THREADS), 0, st, 5, a);
        launches++;
    }
    if (!h->multi) board_stages(nullptr);  // (fid_detect on a multi-dictionary handle is detectMarkers with dictionary 0: no board stage)
    CK(cudaEventRecord(s.ev[ST_D2H], st));
    h->counters[6] += launches;
    CK(cudaGetLastError());
    return FID_OK;
}

static int enqueue_d2h(fid_detector* h, Slot& s, cudaStream_t st, int nf, bool with_pose, bool with_hyp, bool with_board, bool with_charuco, bool with_refine,
                       bool with_diamonds, bool multi = false, bool with_conf = false) {
    const size_t M = (size_t)nf * h->max_markers;
    if (with_conf) CK(cudaMemcpyAsync(s.h_out_conf, s.d_out_conf, sizeof(float) * M, cudaMemcpyDeviceToHost, st));
    if (multi) CK(cudaMemcpyAsync(s.h_out_dict, s.d_out_dict, sizeof(int32_t) * M, cudaMemcpyDeviceToHost, st));
    if (with_diamonds) CK(cudaMemcpyAsync(s.h_dia_n, s.d_dia_n, sizeof(int32_t) * nf, cudaMemcpyDeviceToHost, st));  // collect copies the records
    if (with_refine) {  // counts only: collect copies the lists at their lengths
        CK(cudaMemcpyAsync(s.h_rej_n, s.d_rej_n, sizeof(int32_t) * nf, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(s.h_mr_nrec, s.d_mr_nrec, sizeof(int32_t) * nf, cudaMemcpyDeviceToHost, st));
    }
    CK(cudaMemcpyAsync(s.h_out_count, s.d_out_count, sizeof(int32_t) * nf, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(s.h_out_ids, s.d_out_ids, sizeof(int32_t) * M, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(s.h_out_corners, s.d_out_corners, sizeof(float) * 8 * M, cudaMemcpyDeviceToHost, st));
    if (with_pose) CK(cudaMemcpyAsync(s.h_out_tf, s.d_out_tf, sizeof(fid_transform) * M, cudaMemcpyDeviceToHost, st));
    if (with_hyp) CK(cudaMemcpyAsync(s.h_out_hyp, s.d_out_hyp, sizeof(struct fid_pose_hypotheses) * M, cudaMemcpyDeviceToHost, st));
    if (with_board) CK(cudaMemcpyAsync(s.h_out_board, s.d_out_board, sizeof(fid_board_pose) * nf * h->n_boards, cudaMemcpyDeviceToHost, st));
    if (with_charuco) {
        CK(cudaMemcpyAsync(s.h_out_ch, s.d_out_ch, sizeof(fid_charuco_result) * nf * h->n_charuco, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(s.h_out_ch_ids, s.d_out_ch_ids, sizeof(int32_t) * nf * h->charuco_slots, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(s.h_out_ch_xy, s.d_out_ch_xy, sizeof(float) * 2 * nf * h->charuco_slots, cudaMemcpyDeviceToHost, st));
    }
    CK(cudaMemcpyAsync(s.h_counters, s.d_counters, sizeof(Counters), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(s.h_nsel, s.d_nsel, sizeof(int) * nf, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(s.h_nrawc, s.d_nrawc, sizeof(int) * nf, cudaMemcpyDeviceToHost, st));
    CK(cudaEventRecord(s.ev[ST_COUNT], st));
    CK(cudaEventRecord(s.done, st));
    return FID_OK;
}

static int collect(fid_detector* h, Slot& s, int nf, int max_markers, int32_t* counts, int32_t* ids, float* corners, fid_transform* tfs, bool first_chunk,
                   struct fid_pose_hypotheses* hyps = nullptr, fid_board_pose* boards = nullptr, int ch_first = -1, bool refined = false, bool diamonds = false,
                   int32_t* dict_idx = nullptr, bool multi = false, float* conf = nullptr) {
    CK(cudaEventSynchronize(s.done));
    int status = FID_OK;
    if (diamonds) {  // the diamond records (fid_last_diamonds), each row at the frame with the most diamonds
        int max_d = 0;
        for (int f = 0; f < nf; f++) max_d = std::max(max_d, (int)s.h_dia_n[f]);
        if (max_d) {
            const cudaStream_t st = h->slot_stream[&s - h->slot];
            CK(cudaMemcpy2DAsync(s.h_dia, sizeof(fid_diamond) * max_d, s.d_dia, sizeof(fid_diamond) * FID_MAX_DIAMONDS, sizeof(fid_diamond) * max_d, nf, cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
        }
        for (int f = 0; f < nf; f++) {
            h->last_dia_n.push_back(s.h_dia_n[f]);
            h->last_dia.insert(h->last_dia.end(), s.h_dia + (size_t)f * max_d, s.h_dia + (size_t)f * max_d + s.h_dia_n[f]);
        }
    }
    if (refined) {  // the rejected lists and the recovered markers (fid_last_marker_refinement), each row at the longest frame's length
        const cudaStream_t st = h->slot_stream[&s - h->slot];
        int max_rej = 0, max_rec = 0;
        for (int f = 0; f < nf; f++) {
            max_rej = std::max(max_rej, (int)s.h_rej_n[f]);
            max_rec = std::max(max_rec, (int)s.h_mr_nrec[f]);
        }
        if (max_rej)
            CK(cudaMemcpy2DAsync(s.h_rej, sizeof(float) * 8 * max_rej, s.d_rej, sizeof(float) * 8 * h->max_sel, sizeof(float) * 8 * max_rej, nf, cudaMemcpyDeviceToHost, st));
        if (max_rec) {
            CK(cudaMemcpy2DAsync(s.h_mr_idx, sizeof(int32_t) * max_rec, s.d_mr_idx, sizeof(int32_t) * h->max_markers, sizeof(int32_t) * max_rec, nf, cudaMemcpyDeviceToHost, st));
            CK(cudaMemcpy2DAsync(s.h_mr_board, sizeof(int32_t) * max_rec, s.d_mr_board, sizeof(int32_t) * h->max_markers, sizeof(int32_t) * max_rec, nf, cudaMemcpyDeviceToHost, st));
        }
        CK(cudaStreamSynchronize(st));
        for (int f = 0; f < nf; f++) {
            const int nj = s.h_rej_n[f], nr = s.h_mr_nrec[f];
            h->last_mr_nrej.push_back(nj);
            h->last_mr_nrec.push_back(nr);
            h->last_mr_rej.insert(h->last_mr_rej.end(), s.h_rej + (size_t)f * max_rej * 8, s.h_rej + ((size_t)f * max_rej + nj) * 8);
            h->last_mr_idx.insert(h->last_mr_idx.end(), s.h_mr_idx + (size_t)f * max_rec, s.h_mr_idx + (size_t)f * max_rec + nr);
            h->last_mr_board.insert(h->last_mr_board.end(), s.h_mr_board + (size_t)f * max_rec, s.h_mr_board + (size_t)f * max_rec + nr);
        }
    }
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
        if (hyps) memcpy(hyps + (size_t)f * max_markers, s.h_out_hyp + (size_t)f * h->max_markers, sizeof(struct fid_pose_hypotheses) * n);
        if (dict_idx && multi) memcpy(dict_idx + (size_t)f * max_markers, s.h_out_dict + (size_t)f * h->max_markers, sizeof(int32_t) * n);
        if (dict_idx && !multi) memset(dict_idx + (size_t)f * max_markers, 0, sizeof(int32_t) * n);
        if (conf) memcpy(conf + (size_t)f * max_markers, s.h_out_conf + (size_t)f * h->max_markers, sizeof(float) * n);
    }
    if (boards) memcpy(boards, s.h_out_board, sizeof(fid_board_pose) * nf * h->n_boards);
    if (ch_first >= 0) {  // frames ch_first .. of the ChArUco records of the batch (fid_last_charuco)
        memcpy(h->last_ch.data() + (size_t)ch_first * h->last_ch_n, s.h_out_ch, sizeof(fid_charuco_result) * nf * h->last_ch_n);
        memcpy(h->last_ch_ids.data() + (size_t)ch_first * h->last_ch_slots, s.h_out_ch_ids, sizeof(int32_t) * nf * h->last_ch_slots);
        memcpy(h->last_ch_xy.data() + (size_t)ch_first * h->last_ch_slots * 2, s.h_out_ch_xy, sizeof(float) * 2 * nf * h->last_ch_slots);
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

// The host copy of the records of the batch being returned (fid_last_pose_hypotheses), dense at the caller's max_markers; nullptr
// when the option is off for the batch.
static struct fid_pose_hypotheses* begin_last_hypotheses(fid_detector* h, bool hyp, int n_frames, int max_markers) {
    h->last_hyp_valid = false;
    if (!hyp) return nullptr;
    h->last_hyp_frames = n_frames;
    h->last_hyp_stride = max_markers;
    h->last_hyp.resize((size_t)n_frames * max_markers);
    return h->last_hyp.data();
}
static void end_last_hypotheses(fid_detector* h, bool hyp, const int32_t* counts) {
    if (!hyp) return;
    h->last_hyp_counts.assign(counts, counts + h->last_hyp_frames);
    h->last_hyp_valid = true;
}

// The same for the dictionary indices (fid_last_dict_indices), kept for every batch.
static int32_t* begin_last_dict_indices(fid_detector* h, int n_frames, int max_markers) {
    h->last_di_valid = false;
    h->last_di_frames = n_frames;
    h->last_di_stride = max_markers;
    h->last_di.resize((size_t)n_frames * max_markers);
    return h->last_di.data();
}
static void end_last_dict_indices(fid_detector* h, const int32_t* counts) {
    h->last_di_counts.assign(counts, counts + h->last_di_frames);
    h->last_di_valid = true;
}

// The same for the marker confidences (fid_last_marker_confidence).
static float* begin_last_confidence(fid_detector* h, bool conf, int n_frames, int max_markers) {
    h->last_conf_valid = false;
    if (!conf) return nullptr;
    h->last_conf_frames = n_frames;
    h->last_conf_stride = max_markers;
    h->last_conf.resize((size_t)n_frames * max_markers);
    return h->last_conf.data();
}
static void end_last_confidence(fid_detector* h, bool conf, const int32_t* counts) {
    if (!conf) return;
    h->last_conf_counts.assign(counts, counts + h->last_conf_frames);
    h->last_conf_valid = true;
}

// The same for the board poses (fid_last_board_poses), dense [n_frames][n_boards].
static fid_board_pose* begin_last_boards(fid_detector* h, bool board, int n_frames) {
    h->last_board_valid = false;
    if (!board) return nullptr;
    h->last_board_frames = n_frames;
    h->last_board_n = h->n_boards;
    h->last_board.resize((size_t)n_frames * h->n_boards);
    return h->last_board.data();
}

// The same for the ChArUco records and corners (fid_last_charuco).
static void begin_last_charuco(fid_detector* h, bool ch, int n_frames) {
    h->last_ch_valid = false;
    if (!ch) return;
    h->last_ch_frames = n_frames;
    h->last_ch_n = h->n_charuco;
    h->last_ch_slots = h->charuco_slots;
    h->last_ch.resize((size_t)n_frames * h->n_charuco);
    h->last_ch_ids.resize((size_t)n_frames * h->charuco_slots);
    h->last_ch_xy.resize((size_t)n_frames * h->charuco_slots * 2);
}

// The same for the recovered markers and rejected lists (fid_last_marker_refinement); collect appends frame after frame.
static void begin_last_refinement(fid_detector* h, bool refine, int n_frames) {
    h->last_mr_valid = false;
    if (!refine) return;
    h->last_mr_frames = n_frames;
    h->last_mr_nrec.clear();
    h->last_mr_nrej.clear();
    h->last_mr_idx.clear();
    h->last_mr_board.clear();
    h->last_mr_rej.clear();
}

// The same for the diamonds (fid_last_diamonds); collect appends frame after frame.
static void begin_last_diamonds(fid_detector* h, bool dia, int n_frames) {
    h->last_dia_valid = false;
    if (!dia) return;
    h->last_dia_frames = n_frames;
    h->last_dia_n.clear();
    h->last_dia.clear();
}

// fid_detect_pose_batch; fid_detect (detectMarkers) passes may_refine = false, which also leaves diamonds out.
static int detect_pose_batch(fid_detector* h, int n_frames, const uint8_t* bgr, int bgr_on_device, int width, int height, size_t row_stride, size_t frame_stride,
                             const fid_camera* cam, double fiducial_len, int n_override, const int32_t* override_ids, const double* override_lens,
                             int max_markers, int32_t* counts, int32_t* ids, float* corners, fid_transform* transforms, bool may_refine, bool multi, bool conf) {
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
    const bool hyp = h->pose_hyp && cam;
    struct fid_pose_hypotheses* hyps = begin_last_hypotheses(h, hyp, n_frames, max_markers);
    const bool brd = h->n_boards && cam;
    fid_board_pose* boards = begin_last_boards(h, brd, n_frames);
    const bool chr = h->n_charuco > 0 && multi == h->multi;  // (not fid_detect on a multi-dictionary handle: enqueue_pipeline)
    begin_last_charuco(h, chr, n_frames);
    const bool mr = may_refine && batch_refines(h);
    begin_last_refinement(h, mr, n_frames);
    const bool dia = may_refine && h->diamond.enable;
    begin_last_diamonds(h, dia, n_frames);
    int32_t* dict_idx = begin_last_dict_indices(h, n_frames, max_markers);
    float* confs = begin_last_confidence(h, conf, n_frames, max_markers);
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
            rc = enqueue_pipeline(h, s, cst, nf, g, d_in, cam, fiducial_len, n_override, -1, c > 0 ? &h->slot[(c - 1) % NS] : nullptr, mr, dia, multi, conf);
            if (rc != FID_OK) return rc;
            rc = enqueue_d2h(h, s, cst, nf, cam != nullptr, hyp, brd, chr, mr, dia, multi, conf);
            if (rc != FID_OK) return rc;
            h->last_frames = nf;
        }
        if (c >= NS - 1) {
            const int pc = c - (NS - 1);
            Slot& s = h->slot[pc % NS];
            const int nf = std::min(B, n_frames - pc * B);
            rc = collect(h, s, nf, max_markers, counts + (size_t)pc * B, ids ? ids + (size_t)pc * B * max_markers : nullptr,
                         corners ? corners + (size_t)pc * B * max_markers * 8 : nullptr, (transforms && cam) ? transforms + (size_t)pc * B * max_markers : nullptr, pc == 0,
                         hyps ? hyps + (size_t)pc * B * max_markers : nullptr, boards ? boards + (size_t)pc * B * h->n_boards : nullptr, chr ? pc * B : -1, mr, dia,
                         dict_idx + (size_t)pc * B * max_markers, multi, confs ? confs + (size_t)pc * B * max_markers : nullptr);
            if (rc != FID_OK) status = rc;
        }
    }
    end_last_hypotheses(h, hyp, counts);
    end_last_dict_indices(h, counts);
    end_last_confidence(h, conf, counts);
    h->last_board_valid = brd;
    h->last_ch_valid = chr;
    h->last_mr_valid = mr;
    h->last_dia_valid = dia;
    return status;
}

extern "C" int fid_detect_pose_batch(fid_detector* h, int n_frames, const uint8_t* bgr, int bgr_on_device, int width, int height, size_t row_stride, size_t frame_stride,
                                     const fid_camera* cam, double fiducial_len, int n_override, const int32_t* override_ids, const double* override_lens,
                                     int max_markers, int32_t* counts, int32_t* ids, float* corners, fid_transform* transforms) {
    return detect_pose_batch(h, n_frames, bgr, bgr_on_device, width, height, row_stride, frame_stride, cam, fiducial_len, n_override, override_ids, override_lens,
                             max_markers, counts, ids, corners, transforms, true, h && h->multi, h && h->marker_conf);
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
    const bool mr = batch_refines(h);
    const bool dia = h->diamond.enable != 0;
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
        rc = enqueue_pipeline(h, s, cst, nf, g, d_in, cam, fiducial_len, n_override, -1, prev, mr, dia, h->multi, h->marker_conf != 0);
        if (rc != FID_OK) return rc;
        rc = enqueue_d2h(h, s, cst, nf, cam != nullptr, h->pose_hyp && cam, h->n_boards && cam, h->n_charuco > 0, mr, dia, h->multi, h->marker_conf != 0);
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
    pb.hyp = h->pose_hyp && cam;
    pb.board = h->n_boards && cam;
    pb.charuco = h->n_charuco > 0;
    pb.refine = mr;
    pb.diamonds = dia;
    pb.multi = h->multi;
    pb.conf = h->marker_conf != 0;
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
    struct fid_pose_hypotheses* hyps = begin_last_hypotheses(h, pb.hyp, pb.n_frames, max_markers);
    fid_board_pose* boards = begin_last_boards(h, pb.board, pb.n_frames);
    begin_last_charuco(h, pb.charuco, pb.n_frames);
    begin_last_refinement(h, pb.refine, pb.n_frames);
    begin_last_diamonds(h, pb.diamonds, pb.n_frames);
    int32_t* dict_idx = begin_last_dict_indices(h, pb.n_frames, max_markers);
    float* confs = begin_last_confidence(h, pb.conf, pb.n_frames, max_markers);
    for (int c = 0; c < pb.n_chunks; c++) {
        Slot& s = h->slot[(pb.first_slot + c) % NS];
        const int nf = std::min(B, pb.n_frames - c * B);
        const int rc = collect(h, s, nf, max_markers, counts + (size_t)c * B, ids ? ids + (size_t)c * B * max_markers : nullptr,
                               corners ? corners + (size_t)c * B * max_markers * 8 : nullptr, (transforms && pb.pose) ? transforms + (size_t)c * B * max_markers : nullptr, c == 0,
                               hyps ? hyps + (size_t)c * B * max_markers : nullptr, boards ? boards + (size_t)c * B * h->n_boards : nullptr,
                               pb.charuco ? c * B : -1, pb.refine, pb.diamonds, dict_idx + (size_t)c * B * max_markers, pb.multi,
                               confs ? confs + (size_t)c * B * max_markers : nullptr);
        if (rc != FID_OK) status = rc;
    }
    end_last_hypotheses(h, pb.hyp, counts);
    end_last_dict_indices(h, counts);
    end_last_confidence(h, pb.conf, counts);
    h->last_board_valid = pb.board;
    h->last_ch_valid = pb.charuco;
    h->last_mr_valid = pb.refine;
    h->last_dia_valid = pb.diamonds;
    h->pend_head = (h->pend_head + 1) % MAX_SLOTS;
    h->pend_count--;
    h->slots_in_use -= pb.n_chunks;
    return status;
}

extern "C" int fid_detect(fid_detector* h, const uint8_t* bgr, int width, int height, size_t stride, int max_markers, int* n, int32_t* ids, float* corners) {
    if (!n) return FID_ERR_INVALID_ARG;
    int32_t count = 0;
    const int rc = detect_pose_batch(h, 1, bgr, 0, width, height, stride, stride * (size_t)height, nullptr, 0.0, 0, nullptr, nullptr, max_markers, &count, ids, corners, nullptr, false,
                                     false, false);
    if (rc == FID_OK || rc == FID_ERR_CAPACITY) {
        h->detected = true;
        h->detected_multi = false;
    }
    *n = count;
    return rc;
}

extern "C" int fid_detect_multi_dict(fid_detector* h, const uint8_t* bgr, int width, int height, size_t stride, int max_markers, int* n, int32_t* ids, float* corners,
                                     int32_t* dict_indices) {
    if (!h || !n) return FID_ERR_INVALID_ARG;
    if (h->aruco3.enable) return FID_ERR_UNSUPPORTED;  // the multi-dictionary pass is not pinned with useAruco3Detection
    int32_t count = 0;
    const int rc = detect_pose_batch(h, 1, bgr, 0, width, height, stride, stride * (size_t)height, nullptr, 0.0, 0, nullptr, nullptr, max_markers, &count, ids, corners, nullptr, false,
                                     h->multi, false);
    if (rc == FID_OK || rc == FID_ERR_CAPACITY) {
        h->detected = true;
        h->detected_multi = h->multi;
        if (dict_indices) memcpy(dict_indices, h->last_di.data(), sizeof(int32_t) * count);
    }
    *n = count;
    return rc;
}

extern "C" int fid_last_dict_indices(fid_detector* h, int max_markers, int* n_frames, int32_t* out) {
    if (!h || !n_frames || max_markers < 0 || !h->last_di_valid) return FID_ERR_INVALID_ARG;
    const int nf = h->last_di_frames;
    *n_frames = nf;
    if (!out) return FID_OK;
    for (int f = 0; f < nf; f++)
        if (h->last_di_counts[f] > max_markers) return FID_ERR_CAPACITY;
    for (int f = 0; f < nf; f++) memcpy(out + (size_t)f * max_markers, h->last_di.data() + (size_t)f * h->last_di_stride, sizeof(int32_t) * h->last_di_counts[f]);
    return FID_OK;
}

// Each slot's confidence buffers, allocated by the first use (a failed allocation leaves them for the next use to complete).
static int alloc_confidence(fid_detector* h) {
    CK(cudaSetDevice(h->device));
    const size_t F = h->max_batch, M = F * h->max_markers;
    for (int i = 0; i < h->n_slots; i++) {
        Slot& s = h->slot[i];
        int rc;
        if (!s.d_cand_conf && (rc = dalloc(&s.d_cand_conf, F * h->max_sel)) != FID_OK) return rc;
        if (!s.d_out_conf && (rc = dalloc(&s.d_out_conf, M)) != FID_OK) return rc;
        if (!s.h_out_conf && (rc = halloc(&s.h_out_conf, M)) != FID_OK) return rc;
    }
    return FID_OK;
}

extern "C" int fid_detect_with_confidence(fid_detector* h, const uint8_t* bgr, int width, int height, size_t stride, int max_markers, int* n, int32_t* ids, float* corners,
                                          float* confidence) {
    if (!h || !n) return FID_ERR_INVALID_ARG;
    if (h->multi) return FID_ERR_UNSUPPORTED;  // cv2 has no confidence for detectMarkersMultiDict
    if (h->pend_count) return FID_ERR_INVALID_ARG;
    int rc = alloc_confidence(h);
    if (rc != FID_OK) return rc;
    int32_t count = 0;
    rc = detect_pose_batch(h, 1, bgr, 0, width, height, stride, stride * (size_t)height, nullptr, 0.0, 0, nullptr, nullptr, max_markers, &count, ids, corners, nullptr, false, false,
                           true);
    if (rc == FID_OK || rc == FID_ERR_CAPACITY) {
        h->detected = true;
        h->detected_multi = false;
        if (confidence) memcpy(confidence, h->last_conf.data(), sizeof(float) * count);
    }
    *n = count;
    return rc;
}

extern "C" int fid_set_marker_confidence(fid_detector* h, int enable) {
    if (!h || h->pend_count) return FID_ERR_INVALID_ARG;  // batches in flight were enqueued with the old setting
    if (enable && (h->multi || h->batch_refine)) return FID_ERR_UNSUPPORTED;  // neither detectMarkersMultiDict nor recovered markers have a confidence
    if (enable) {
        const int rc = alloc_confidence(h);
        if (rc != FID_OK) return rc;
    }
    h->marker_conf = enable ? 1 : 0;
    return FID_OK;
}

// detectInvertedMarker.  Slot 0's candidates (fid_debug_rejected) came from the other mode once the setting changes.
extern "C" int fid_set_detect_inverted_marker(fid_detector* h, int enable) {
    if (!h || h->pend_count) return FID_ERR_INVALID_ARG;  // batches in flight were enqueued with the old setting
    if (enable && (h->batch_refine || h->mrefine.enable)) return FID_ERR_UNSUPPORTED;  // refineDetectedMarkers under the flag is not modelled
    const int v = enable ? 1 : 0;
    if (v != h->inverted) h->detected = false;
    h->inverted = v;
    return FID_OK;
}

extern "C" int fid_last_marker_confidence(fid_detector* h, int max_markers, int* n_frames, float* out) {
    if (!h || !n_frames || max_markers < 0 || !h->last_conf_valid) return FID_ERR_INVALID_ARG;
    const int nf = h->last_conf_frames;
    *n_frames = nf;
    if (!out) return FID_OK;
    for (int f = 0; f < nf; f++)
        if (h->last_conf_counts[f] > max_markers) return FID_ERR_CAPACITY;
    for (int f = 0; f < nf; f++) memcpy(out + (size_t)f * max_markers, h->last_conf.data() + (size_t)f * h->last_conf_stride, sizeof(float) * h->last_conf_counts[f]);
    return FID_OK;
}

// Bytes of one frame's pyramid levels 1.. and segmentation plane that any frame up to max_w x max_h needs under the parameters p.
// The levels grow with the frame.  The plane's width is round(fxfy * W') with fxfy = m / (m + max(W', H') r) <= m / (m + W' r), and
// m W' / (m + W' r) grows with W', so max_w bounds it (+ 2 for the float32 rounding of fxfy and of the product); the same for the height.
// With r = 0, fxfy = 1 and the gray plane serves as the segmentation plane.
static void a3_plane_bytes(const fid_detector* h, const fid_aruco3_params& p, size_t* pyr, size_t* seg) {
    A3Geom g;
    a3_geometry(h->max_w, h->max_h, p.minSideLengthCanonicalImg, p.minMarkerLengthRatioOriginalImg, &g);
    *pyr = g.pyr_frame_bytes;
    *seg = 0;
    if (p.minMarkerLengthRatioOriginalImg > 0) {
        const double m = p.minSideLengthCanonicalImg, r = p.minMarkerLengthRatioOriginalImg;
        const size_t w = std::min<size_t>(h->max_w, (size_t)(m * h->max_w / (m + h->max_w * r)) + 2);
        const size_t ht = std::min<size_t>(h->max_h, (size_t)(m * h->max_h / (m + h->max_h * r)) + 2);
        *seg = w * ht;
    }
}

extern "C" int fid_set_aruco3(fid_detector* h, const fid_aruco3_params* params) {
    if (!h || !params || h->pend_count) return FID_ERR_INVALID_ARG;  // batches in flight were enqueued with the old setting
    const fid_aruco3_params p = *params;
    if (p.enable) {
        if (p.minSideLengthCanonicalImg < 1 || p.minSideLengthCanonicalImg > 16384 || !(p.minMarkerLengthRatioOriginalImg >= 0.0 && p.minMarkerLengthRatioOriginalImg <= 1.0))
            return FID_ERR_INVALID_ARG;
        if (h->multi || h->batch_refine) return FID_ERR_UNSUPPORTED;
        CK(cudaSetDevice(h->device));
        size_t pyr, seg;
        a3_plane_bytes(h, p, &pyr, &seg);
        const size_t F = h->max_batch;
        for (int i = 0; i < h->n_slots; i++) CK(cudaStreamSynchronize(h->slot_stream[i]));
        CK(cudaStreamSynchronize(h->stream));
        int rc;
        for (int i = 0; i < h->n_slots; i++) {  // grown, never shrunk (a failed allocation leaves the mode as it was; the next enable completes it)
            Slot& s = h->slot[i];
            if (F * pyr > s.a3_pyr_cap) {
                if (s.d_a3_pyr) cudaFree(s.d_a3_pyr);
                s.d_a3_pyr = nullptr;
                s.a3_pyr_cap = 0;
                if ((rc = dalloc(&s.d_a3_pyr, F * pyr)) != FID_OK) return rc;
                s.a3_pyr_cap = F * pyr;
            }
            if (F * seg > s.a3_seg_cap) {
                if (s.d_a3_seg) cudaFree(s.d_a3_seg);
                s.d_a3_seg = nullptr;
                s.a3_seg_cap = 0;
                if ((rc = dalloc(&s.d_a3_seg, F * seg)) != FID_OK) return rc;
                s.a3_seg_cap = F * seg;
            }
        }
    }
    h->aruco3 = p;
    return FID_OK;
}

extern "C" int fid_debug_aruco3_planes(fid_detector* h, const uint8_t* bgr, int width, int height, size_t stride, int32_t* info, uint8_t* seg, uint8_t* pyramid,
                                       size_t pyramid_bytes) {
    if (!h || !bgr || !info || width < 16 || height < 16 || width > h->max_w || height > h->max_h || stride < (size_t)width * h->bpp) return FID_ERR_INVALID_ARG;
    if (h->pend_count || !h->aruco3.enable) return FID_ERR_INVALID_ARG;  // slot 0 may belong to a batch in flight
    A3Geom ag;
    if (!a3_geometry(width, height, h->aruco3.minSideLengthCanonicalImg, h->aruco3.minMarkerLengthRatioOriginalImg, &ag)) return FID_ERR_INVALID_ARG;
    info[0] = ag.seg_w;
    info[1] = ag.seg_h;
    info[2] = ag.n_levels;
    info[3] = ag.closest;
    if (!seg && !pyramid) return FID_OK;  // sizes only
    if (pyramid && pyramid_bytes < ag.pyr_frame_bytes) return FID_ERR_CAPACITY;
    CK(cudaSetDevice(h->device));
    Slot& s = h->slot[0];
    CK(cudaMemcpy2DAsync(s.d_bgr, (size_t)width * h->bpp, bgr, stride, (size_t)width * h->bpp, height, cudaMemcpyHostToDevice, h->stream));
    const FrameGeom g = make_geom(h, width, height, (size_t)width * h->bpp, (size_t)width * h->bpp * height);
    enqueue_aruco3_planes(h, s, h->stream, 1, g, s.d_bgr, ag);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(h->stream));
    if (seg) {
        if (ag.resized)
            CK(cudaMemcpy(seg, s.d_a3_seg, (size_t)ag.seg_w * ag.seg_h, cudaMemcpyDeviceToHost));
        else
            CK(cudaMemcpy2D(seg, width, s.d_gray, g.gray_pitch, width, height, cudaMemcpyDeviceToHost));
    }
    if (pyramid && ag.pyr_frame_bytes) CK(cudaMemcpy(pyramid, s.d_a3_pyr, ag.pyr_frame_bytes, cudaMemcpyDeviceToHost));
    return FID_OK;
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

extern "C" int fid_set_pose_hypotheses(fid_detector* h, int enable) {
    if (!h || h->pend_count) return FID_ERR_INVALID_ARG;  // batches in flight were enqueued with the old setting
    if (enable) {  // (a failed allocation leaves the option off; the next enable completes it)
        CK(cudaSetDevice(h->device));
        const size_t M = (size_t)h->max_batch * h->max_markers;
        for (int i = 0; i < h->n_slots; i++) {
            Slot& s = h->slot[i];
            int rc;
            if (!s.d_out_hyp && (rc = dalloc(&s.d_out_hyp, M)) != FID_OK) return rc;
            if (!s.h_out_hyp && (rc = halloc(&s.h_out_hyp, M)) != FID_OK) return rc;
        }
    }
    h->pose_hyp = enable ? 1 : 0;
    return FID_OK;
}

extern "C" int fid_pose_hypotheses(fid_detector* h, int n, const int32_t* ids, const float* corners, const fid_camera* cam, double fiducial_len, int n_override,
                                   const int32_t* override_ids, const double* override_lens, struct fid_pose_hypotheses* out) {
    if (!h || n < 0 || n > 4096 || !cam || !(fiducial_len > 0) || (n > 0 && (!ids || !corners || !out))) return FID_ERR_INVALID_ARG;
    if (h->pend_count) return FID_ERR_INVALID_ARG;  // batches in flight read the shared override table
    if (n == 0) return FID_OK;
    CK(cudaSetDevice(h->device));
    int rc = upload_overrides(h, n_override, override_ids, override_lens);
    if (rc != FID_OK) return rc;
    if (!h->d_hyp_list && (rc = dalloc(&h->d_hyp_list, 4096)) != FID_OK) return rc;
    CK(cudaMemcpyAsync(h->d_pose_ids, ids, sizeof(int32_t) * n, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(h->d_pose_corners, corners, sizeof(float) * 8 * n, cudaMemcpyHostToDevice, h->stream));
    PoseHypListArgs a{};
    a.n = n;
    a.ids = h->d_pose_ids;
    a.corners = h->d_pose_corners;
    a.cam = make_camera(cam);
    a.fiducial_len = fiducial_len;
    a.n_override = n_override;
    a.override_ids = h->d_override_ids;
    a.override_lens = h->d_override_lens;
    a.out = h->d_hyp_list;
    k_pose_hypotheses_list<<<(n + 63) / 64, 64, 0, h->stream>>>(a);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(out, h->d_hyp_list, sizeof(struct fid_pose_hypotheses) * n, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return FID_OK;
}

extern "C" int fid_last_pose_hypotheses(fid_detector* h, int max_markers, int* n_frames, struct fid_pose_hypotheses* out) {
    if (!h || !n_frames || max_markers < 0 || !h->last_hyp_valid) return FID_ERR_INVALID_ARG;
    const int nf = h->last_hyp_frames;
    *n_frames = nf;
    if (!out) return FID_OK;
    for (int f = 0; f < nf; f++)
        if (h->last_hyp_counts[f] > max_markers) return FID_ERR_CAPACITY;
    for (int f = 0; f < nf; f++)
        memcpy(out + (size_t)f * max_markers, h->last_hyp.data() + (size_t)f * h->last_hyp_stride, sizeof(struct fid_pose_hypotheses) * h->last_hyp_counts[f]);
    return FID_OK;
}

// Validates a family list (fid_set_family_*): every index must name an entry of the handle's dictionary list.
static bool families_valid(const fid_detector* h, int n, const int32_t* family) {
    if (n > 0 && !family) return false;
    for (int i = 0; i < n; i++)
        if (family[i] < 0 || family[i] >= h->n_dicts) return false;
    return true;
}

// fid_set_boards (family = nullptr: no family, refused in multi-dictionary mode) and fid_set_family_boards
static int set_boards(fid_detector* h, int n_boards, const fid_board* boards, const int32_t* family) {
    if (!h || h->pend_count) return FID_ERR_INVALID_ARG;  // batches in flight read the board tables
    if (n_boards < 0 || n_boards > FID_MAX_BOARDS || (n_boards > 0 && !boards)) return FID_ERR_INVALID_ARG;
    if (family && !families_valid(h, n_boards, family)) return FID_ERR_INVALID_ARG;
    if (n_boards > 0 && h->multi && !family) return FID_ERR_UNSUPPORTED;  // a board without a family is ambiguous with several dictionaries
    std::vector<int32_t> off(1, 0), keys, marker;
    std::vector<float> obj;
    for (int b = 0; b < n_boards; b++) {
        const fid_board& B = boards[b];
        if (B.n_markers < 1 || B.n_markers > 4096 || !B.ids || !B.obj_points) return FID_ERR_INVALID_ARG;
        for (int i = 0; i < B.n_markers * 12; i++)
            if (!std::isfinite(B.obj_points[i])) return FID_ERR_INVALID_ARG;
        std::vector<int32_t> ord(B.n_markers);
        for (int i = 0; i < B.n_markers; i++) ord[i] = i;
        std::sort(ord.begin(), ord.end(), [&](int x, int y) { return B.ids[x] < B.ids[y]; });
        for (int i = 0; i < B.n_markers; i++) {
            if (i > 0 && B.ids[ord[i]] == B.ids[ord[i - 1]]) return FID_ERR_INVALID_ARG;  // a repeated id within one board
            keys.push_back(B.ids[ord[i]]);
            marker.push_back(ord[i]);
        }
        obj.insert(obj.end(), B.obj_points, B.obj_points + (size_t)B.n_markers * 12);
        off.push_back((int32_t)keys.size());
    }
    CK(cudaSetDevice(h->device));
    for (void* p : {(void*)h->d_board_off, (void*)h->d_board_keys, (void*)h->d_board_marker, (void*)h->d_board_obj})
        if (p) cudaFree(p);
    h->d_board_off = h->d_board_keys = h->d_board_marker = nullptr;
    h->d_board_obj = nullptr;
    h->n_boards = 0;
    if (n_boards == 0) return FID_OK;
    int rc;
    const size_t M = (size_t)h->max_batch * FID_MAX_BOARDS;
    for (int i = 0; i < h->n_slots; i++) {  // (a failed allocation leaves the boards off; the next call completes it)
        Slot& s = h->slot[i];
        if (!s.d_out_board && (rc = dalloc(&s.d_out_board, M)) != FID_OK) return rc;
        if (!s.h_out_board && (rc = halloc(&s.h_out_board, M)) != FID_OK) return rc;
    }
    if (!h->d_board_list && (rc = dalloc(&h->d_board_list, FID_MAX_BOARDS)) != FID_OK) return rc;
    if (!h->d_board_count && (rc = dalloc(&h->d_board_count, 1)) != FID_OK) return rc;
    if ((rc = dalloc(&h->d_board_off, off.size())) != FID_OK || (rc = dalloc(&h->d_board_keys, keys.size())) != FID_OK ||
        (rc = dalloc(&h->d_board_marker, marker.size())) != FID_OK || (rc = dalloc(&h->d_board_obj, obj.size())) != FID_OK)
        return rc;
    CK(cudaMemcpy(h->d_board_off, off.data(), sizeof(int32_t) * off.size(), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(h->d_board_keys, keys.data(), sizeof(int32_t) * keys.size(), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(h->d_board_marker, marker.data(), sizeof(int32_t) * marker.size(), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(h->d_board_obj, obj.data(), sizeof(float) * obj.size(), cudaMemcpyHostToDevice));
    for (int b = 0; b < n_boards; b++) h->board_fam[b] = family ? family[b] : 0;
    h->board_bound = family != nullptr;
    h->n_boards = n_boards;
    return FID_OK;
}

extern "C" int fid_set_boards(fid_detector* h, int n_boards, const fid_board* boards) { return set_boards(h, n_boards, boards, nullptr); }

extern "C" int fid_set_family_boards(fid_detector* h, int n_boards, const fid_board* boards, const int32_t* dict_index) {
    if (!dict_index) return FID_ERR_INVALID_ARG;
    return set_boards(h, n_boards, boards, dict_index);
}

extern "C" int fid_estimate_board_poses(fid_detector* h, int n, const int32_t* ids, const float* corners, const fid_camera* cam, fid_board_pose* out) {
    if (!h || n < 0 || n > FID_MAX_MARKERS || !cam || !out || (n > 0 && (!ids || !corners)) || h->n_boards == 0) return FID_ERR_INVALID_ARG;
    if (h->multi) return FID_ERR_UNSUPPORTED;  // the list carries no family: the batch calls serve this mode
    CK(cudaSetDevice(h->device));
    if (n > 0) {
        CK(cudaMemcpyAsync(h->d_pose_ids, ids, sizeof(int32_t) * n, cudaMemcpyHostToDevice, h->stream));
        CK(cudaMemcpyAsync(h->d_pose_corners, corners, sizeof(float) * 8 * n, cudaMemcpyHostToDevice, h->stream));
    }
    CK(cudaMemcpyAsync(h->d_board_count, &n, sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
    k_board_pose<<<h->n_boards, FID_BOARD_LANES, 0, h->stream>>>(board_args(h, h->d_board_count, h->d_pose_ids, h->d_pose_corners, n, cam, h->d_board_list));
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(out, h->d_board_list, sizeof(fid_board_pose) * h->n_boards, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return FID_OK;
}

extern "C" int fid_last_board_poses(fid_detector* h, int max_boards, int* n_frames, int* n_boards, fid_board_pose* out) {
    if (!h || !n_frames || !n_boards || max_boards < 0 || !h->last_board_valid) return FID_ERR_INVALID_ARG;
    const int nf = h->last_board_frames, nb = h->last_board_n;
    *n_frames = nf;
    *n_boards = nb;
    if (!out) return FID_OK;
    if (max_boards < nb) return FID_ERR_CAPACITY;
    for (int f = 0; f < nf; f++) memcpy(out + (size_t)f * max_boards, h->last_board.data() + (size_t)f * nb, sizeof(fid_board_pose) * nb);
    return FID_OK;
}

// fid_set_charuco_boards (family = nullptr) and fid_set_family_charuco_boards, as set_boards
static int set_charuco_boards(fid_detector* h, int n_boards, const fid_charuco_board* boards, const int32_t* family) {
    if (!h || h->pend_count) return FID_ERR_INVALID_ARG;  // batches in flight read the board tables
    if (n_boards < 0 || n_boards > FID_MAX_CHARUCO_BOARDS || (n_boards > 0 && !boards)) return FID_ERR_INVALID_ARG;
    if (family && !families_valid(h, n_boards, family)) return FID_ERR_INVALID_ARG;
    if (n_boards > 0 && h->multi && !family) return FID_ERR_UNSUPPORTED;
    std::vector<CharucoBoardDev> bd;
    std::vector<int32_t> keys, marker, ids, near_n, near_idx, near_corner;
    std::vector<float> obj, chess;
    for (int b = 0; b < n_boards; b++) {
        const fid_charuco_board& C = boards[b];
        const int sx = C.squares_x, sy = C.squares_y;
        if (sx < 2 || sy < 2 || sx > FID_MAX_CHARUCO_CORNERS + 1 || sy > FID_MAX_CHARUCO_CORNERS + 1 || (sx - 1) * (sy - 1) > FID_MAX_CHARUCO_CORNERS) return FID_ERR_INVALID_ARG;
        if (!(C.square_length > 0) || !(C.marker_length > 0) || !(C.marker_length < C.square_length) || !std::isfinite(C.square_length)) return FID_ERR_INVALID_ARG;
        if (C.min_markers < 0 || C.min_markers > 2) return FID_ERR_INVALID_ARG;  // cv2 asserts outside 0..2
        const int nm = charuco_n_markers(sx, sy), nc = charuco_n_corners(sx, sy);
        if (nm > h->dict_P[family ? family[b] : 0].n_markers) return FID_ERR_INVALID_ARG;  // more markers than the dictionary has
        CharucoBoardDev d{nm, nc, (int)ids.size(), (int)near_n.size(), C.min_markers, C.check_markers ? 1 : 0, family ? family[b] : 0};
        std::vector<int32_t> bid(nm);
        for (int i = 0; i < nm; i++) bid[i] = C.ids ? C.ids[i] : i;
        std::vector<int32_t> ord(nm);
        for (int i = 0; i < nm; i++) ord[i] = i;
        std::sort(ord.begin(), ord.end(), [&](int x, int y) { return bid[x] < bid[y]; });
        for (int i = 0; i < nm; i++) {
            if (i > 0 && bid[ord[i]] == bid[ord[i - 1]]) return FID_ERR_INVALID_ARG;  // a repeated id within one board
            keys.push_back(bid[ord[i]]);
            marker.push_back(ord[i]);
        }
        ids.insert(ids.end(), bid.begin(), bid.end());
        const size_t o0 = obj.size(), c0 = chess.size(), n0 = near_n.size();
        obj.resize(o0 + (size_t)nm * 12);
        chess.resize(c0 + (size_t)nc * 3);
        near_n.resize(n0 + nc);
        near_idx.resize(2 * (n0 + nc));
        near_corner.resize(2 * (n0 + nc));
        if (!charuco_layout(sx, sy, C.square_length, C.marker_length, C.legacy_pattern != 0, obj.data() + o0, chess.data() + c0, near_n.data() + n0,
                            near_idx.data() + 2 * n0, near_corner.data() + 2 * n0))
            return FID_ERR_INVALID_ARG;
        bd.push_back(d);
    }
    CK(cudaSetDevice(h->device));
    CK(cudaDeviceSynchronize());
    for (void* p : {(void*)h->d_ch_boards, (void*)h->d_ch_keys, (void*)h->d_ch_marker, (void*)h->d_ch_ids, (void*)h->d_ch_near_n, (void*)h->d_ch_near_idx,
                    (void*)h->d_ch_near_corner, (void*)h->d_ch_obj, (void*)h->d_ch_chess})
        if (p) cudaFree(p);
    h->d_ch_boards = nullptr;
    h->d_ch_keys = h->d_ch_marker = h->d_ch_ids = h->d_ch_near_n = h->d_ch_near_idx = h->d_ch_near_corner = nullptr;
    h->d_ch_obj = h->d_ch_chess = nullptr;
    h->n_charuco = 0;
    h->charuco_slots = 0;
    if (n_boards == 0) return FID_OK;
    const int slots = (int)near_n.size();
    int rc;
    for (int i = 0; i < h->n_slots; i++) {  // (a failed allocation leaves the boards off; the next call completes it)
        Slot& s = h->slot[i];
        if (!s.d_out_ch && (rc = dalloc(&s.d_out_ch, (size_t)h->max_batch * FID_MAX_CHARUCO_BOARDS)) != FID_OK) return rc;
        if (!s.h_out_ch && (rc = halloc(&s.h_out_ch, (size_t)h->max_batch * FID_MAX_CHARUCO_BOARDS)) != FID_OK) return rc;
        if (s.ch_slot_cap < slots) {
            for (void* p : {(void*)s.d_out_ch_ids, (void*)s.d_out_ch_xy})
                if (p) cudaFree(p);
            for (void* p : {(void*)s.h_out_ch_ids, (void*)s.h_out_ch_xy})
                if (p) cudaFreeHost(p);
            s.d_out_ch_ids = nullptr;
            s.d_out_ch_xy = s.h_out_ch_xy = nullptr;
            s.h_out_ch_ids = nullptr;
            s.ch_slot_cap = 0;
            const size_t M = (size_t)h->max_batch * slots;
            if ((rc = dalloc(&s.d_out_ch_ids, M)) != FID_OK || (rc = dalloc(&s.d_out_ch_xy, 2 * M)) != FID_OK || (rc = halloc(&s.h_out_ch_ids, M)) != FID_OK ||
                (rc = halloc(&s.h_out_ch_xy, 2 * M)) != FID_OK)
                return rc;
            s.ch_slot_cap = slots;
        }
    }
    if (!h->d_ch_masks) {
        std::vector<float> masks(FID_CHARUCO_MASK_FLOATS);
        charuco_subpix_masks(masks.data());
        if ((rc = dalloc(&h->d_ch_masks, masks.size())) != FID_OK) return rc;
        CK(cudaMemcpy(h->d_ch_masks, masks.data(), sizeof(float) * masks.size(), cudaMemcpyHostToDevice));
        CK(cudaFuncSetAttribute(k_charuco, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CHARUCO_SMEM));
    }
    if (!h->d_ch_count && (rc = dalloc(&h->d_ch_count, 1)) != FID_OK) return rc;
    if (!h->d_ch_list && (rc = dalloc(&h->d_ch_list, FID_MAX_CHARUCO_BOARDS)) != FID_OK) return rc;
    if (h->d_ch_list_ids) cudaFree(h->d_ch_list_ids);
    if (h->d_ch_list_xy) cudaFree(h->d_ch_list_xy);
    h->d_ch_list_ids = nullptr;
    h->d_ch_list_xy = nullptr;
    if ((rc = dalloc(&h->d_ch_list_ids, (size_t)slots)) != FID_OK || (rc = dalloc(&h->d_ch_list_xy, (size_t)2 * slots)) != FID_OK) return rc;
    if ((rc = dalloc(&h->d_ch_boards, bd.size())) != FID_OK || (rc = dalloc(&h->d_ch_keys, keys.size())) != FID_OK || (rc = dalloc(&h->d_ch_marker, marker.size())) != FID_OK ||
        (rc = dalloc(&h->d_ch_ids, ids.size())) != FID_OK || (rc = dalloc(&h->d_ch_near_n, near_n.size())) != FID_OK ||
        (rc = dalloc(&h->d_ch_near_idx, near_idx.size())) != FID_OK || (rc = dalloc(&h->d_ch_near_corner, near_corner.size())) != FID_OK ||
        (rc = dalloc(&h->d_ch_obj, obj.size())) != FID_OK || (rc = dalloc(&h->d_ch_chess, chess.size())) != FID_OK)
        return rc;
    CK(cudaMemcpy(h->d_ch_boards, bd.data(), sizeof(CharucoBoardDev) * bd.size(), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(h->d_ch_keys, keys.data(), sizeof(int32_t) * keys.size(), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(h->d_ch_marker, marker.data(), sizeof(int32_t) * marker.size(), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(h->d_ch_ids, ids.data(), sizeof(int32_t) * ids.size(), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(h->d_ch_near_n, near_n.data(), sizeof(int32_t) * near_n.size(), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(h->d_ch_near_idx, near_idx.data(), sizeof(int32_t) * near_idx.size(), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(h->d_ch_near_corner, near_corner.data(), sizeof(int32_t) * near_corner.size(), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(h->d_ch_obj, obj.data(), sizeof(float) * obj.size(), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(h->d_ch_chess, chess.data(), sizeof(float) * chess.size(), cudaMemcpyHostToDevice));
    for (int b = 0; b < n_boards; b++) {
        h->charuco_fam[b] = family ? family[b] : 0;
        h->charuco_nm[b] = bd[b].n_markers;
    }
    h->charuco_bound = family != nullptr;
    h->n_charuco = n_boards;
    h->charuco_slots = slots;
    return FID_OK;
}

extern "C" int fid_set_charuco_boards(fid_detector* h, int n_boards, const fid_charuco_board* boards) { return set_charuco_boards(h, n_boards, boards, nullptr); }

extern "C" int fid_set_family_charuco_boards(fid_detector* h, int n_boards, const fid_charuco_board* boards, const int32_t* dict_index) {
    if (!dict_index) return FID_ERR_INVALID_ARG;
    return set_charuco_boards(h, n_boards, boards, dict_index);
}

extern "C" int fid_detect_charuco(fid_detector* h, const uint8_t* bgr, int width, int height, size_t stride, int n, const int32_t* ids, const float* corners,
                                  const fid_camera* cam, fid_charuco_result* results, int32_t* corner_ids, float* corner_xy) {
    if (!h || !bgr || n < 0 || n > FID_MAX_MARKERS || (n > 0 && (!ids || !corners)) || !results || !corner_ids || !corner_xy || h->n_charuco == 0) return FID_ERR_INVALID_ARG;
    if (h->multi) return FID_ERR_UNSUPPORTED;  // the list carries no family: the batch calls serve this mode
    if (width < 16 || height < 16 || width > h->max_w || height > h->max_h || stride < (size_t)width * h->bpp) return FID_ERR_INVALID_ARG;
    if (h->pend_count) return FID_ERR_INVALID_ARG;  // slot 0 may belong to a batch in flight
    CK(cudaSetDevice(h->device));
    Slot& s = h->slot[0];
    CK(cudaMemcpy2DAsync(s.d_bgr, (size_t)width * h->bpp, bgr, stride, (size_t)width * h->bpp, height, cudaMemcpyHostToDevice, h->stream));
    if (n > 0) {
        CK(cudaMemcpyAsync(h->d_pose_ids, ids, sizeof(int32_t) * n, cudaMemcpyHostToDevice, h->stream));
        CK(cudaMemcpyAsync(h->d_pose_corners, corners, sizeof(float) * 8 * n, cudaMemcpyHostToDevice, h->stream));
    }
    CK(cudaMemcpyAsync(h->d_ch_count, &n, sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
    k_charuco<<<h->n_charuco, CHARUCO_THREADS, CHARUCO_SMEM, h->stream>>>(charuco_args(h, s.d_bgr, (size_t)width * h->bpp, (size_t)width * h->bpp * height, width, height,
                                                                                      h->d_ch_count, h->d_pose_ids, h->d_pose_corners, FID_MAX_MARKERS, cam, h->d_ch_list,
                                                                                      h->d_ch_list_ids, h->d_ch_list_xy));
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(results, h->d_ch_list, sizeof(fid_charuco_result) * h->n_charuco, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaMemcpyAsync(corner_ids, h->d_ch_list_ids, sizeof(int32_t) * h->charuco_slots, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaMemcpyAsync(corner_xy, h->d_ch_list_xy, sizeof(float) * 2 * h->charuco_slots, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return FID_OK;
}

extern "C" int fid_last_charuco(fid_detector* h, int max_slots, int* n_frames, int* n_boards, int* n_slots, fid_charuco_result* results, int32_t* corner_ids,
                                float* corner_xy) {
    if (!h || !n_frames || !n_boards || !n_slots || max_slots < 0 || !h->last_ch_valid) return FID_ERR_INVALID_ARG;
    const int nf = h->last_ch_frames, nb = h->last_ch_n, ns = h->last_ch_slots;
    *n_frames = nf;
    *n_boards = nb;
    *n_slots = ns;
    if (!results) return FID_OK;
    if (!corner_ids || !corner_xy) return FID_ERR_INVALID_ARG;
    if (max_slots < ns) return FID_ERR_CAPACITY;
    memcpy(results, h->last_ch.data(), sizeof(fid_charuco_result) * nf * nb);
    for (int f = 0; f < nf; f++) {
        memcpy(corner_ids + (size_t)f * max_slots, h->last_ch_ids.data() + (size_t)f * ns, sizeof(int32_t) * ns);
        memcpy(corner_xy + (size_t)f * max_slots * 2, h->last_ch_xy.data() + (size_t)f * ns * 2, sizeof(float) * 2 * ns);
    }
    return FID_OK;
}

extern "C" int fid_set_marker_refinement(fid_detector* h, const fid_marker_refine_params* params) {
    if (!h || !params || h->pend_count) return FID_ERR_INVALID_ARG;
    const fid_marker_refine_params p = *params;
    if (p.enable && (!(p.min_rep_distance > 0) || !std::isfinite(p.min_rep_distance) || !std::isfinite(p.error_correction_rate))) return FID_ERR_INVALID_ARG;
    if (p.enable && h->inverted) return FID_ERR_UNSUPPORTED;  // refineDetectedMarkers with detectInvertedMarker is not modelled
    if (p.enable) {  // (a failed allocation leaves the option off; the next enable completes it)
        CK(cudaSetDevice(h->device));
        int rc;
        if (!h->d_mr_i && (rc = dalloc(&h->d_mr_i, 4 + 3 * (size_t)FID_MAX_MARKERS)) != FID_OK) return rc;
        if (!h->d_mr_f && (rc = dalloc(&h->d_mr_f, 8 * ((size_t)FID_MAX_MARKERS + FID_MAX_REJECTED))) != FID_OK) return rc;
        CK(cudaFuncSetAttribute(k_marker_refine, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)MREFINE_SMEM));
    }
    h->mrefine = p;
    h->mrefine.enable = p.enable ? 1 : 0;
    return FID_OK;
}

extern "C" int fid_refine_detected_markers(fid_detector* h, const uint8_t* bgr, int width, int height, size_t stride, int n, int32_t* ids, float* corners,
                                           int max_markers, int n_rejected, const float* rejected, const fid_camera* cam, int* n_out, int32_t* recovered_idx,
                                           int32_t* recovered_board) {
    if (!h || !bgr || !n_out || !recovered_idx || !recovered_board || max_markers < 0 || max_markers > FID_MAX_MARKERS || n < 0 || n > max_markers ||
        (max_markers > 0 && (!ids || !corners)) || n_rejected < 0 || n_rejected > FID_MAX_REJECTED || (n_rejected > 0 && !rejected))
        return FID_ERR_INVALID_ARG;
    if (width < 16 || height < 16 || width > h->max_w || height > h->max_h || stride < (size_t)width * h->bpp) return FID_ERR_INVALID_ARG;
    if (h->inverted) return FID_ERR_UNSUPPORTED;  // refineDetectedMarkers with detectInvertedMarker is not modelled
    if (!h->mrefine.enable || h->n_boards + h->n_charuco == 0) return FID_ERR_INVALID_ARG;
    if (h->multi) return FID_ERR_UNSUPPORTED;  // the lists carry no family
    if (h->pend_count) return FID_ERR_INVALID_ARG;  // slot 0 may belong to a batch in flight
    CK(cudaSetDevice(h->device));
    Slot& s = h->slot[0];
    int32_t* d_count = h->d_mr_i;
    int32_t* d_ids = h->d_mr_i + 4;
    int32_t* d_rec_idx = d_ids + FID_MAX_MARKERS;
    int32_t* d_rec_board = d_rec_idx + FID_MAX_MARKERS;
    float* d_corners = h->d_mr_f;
    float* d_rej = h->d_mr_f + 8 * FID_MAX_MARKERS;
    const int32_t head[4] = {n, n_rejected, 0, 0};
    CK(cudaMemcpy2DAsync(s.d_bgr, (size_t)width * h->bpp, bgr, stride, (size_t)width * h->bpp, height, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(d_count, head, sizeof(head), cudaMemcpyHostToDevice, h->stream));
    if (n > 0) {
        CK(cudaMemcpyAsync(d_ids, ids, sizeof(int32_t) * n, cudaMemcpyHostToDevice, h->stream));
        CK(cudaMemcpyAsync(d_corners, corners, sizeof(float) * 8 * n, cudaMemcpyHostToDevice, h->stream));
    }
    if (n_rejected > 0) CK(cudaMemcpyAsync(d_rej, rejected, sizeof(float) * 8 * n_rejected, cudaMemcpyHostToDevice, h->stream));
    MarkerRefineArgs a = marker_refine_args(h, s.d_bgr, (size_t)width * h->bpp, (size_t)width * h->bpp * height, width, height, cam);
    a.n_rej = d_count + 1;
    a.rej = d_rej;
    a.max_rej = FID_MAX_REJECTED;
    a.max_markers = max_markers;
    a.count = d_count;
    a.ids = d_ids;
    a.corners = d_corners;
    a.n_rec = d_count + 2;
    a.rec_idx = d_rec_idx;
    a.rec_board = d_rec_board;
    a.overflow = reinterpret_cast<uint32_t*>(d_count + 3);
    k_marker_refine<<<1, MREFINE_THREADS, MREFINE_SMEM, h->stream>>>(a);
    CK(cudaGetLastError());
    int32_t out[4];
    CK(cudaMemcpyAsync(out, d_count, sizeof(out), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    if (out[3]) return FID_ERR_CAPACITY;
    const int nr = out[2];
    if (nr > 0) {
        CK(cudaMemcpy(ids + n, d_ids + n, sizeof(int32_t) * nr, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(corners + (size_t)8 * n, d_corners + (size_t)8 * n, sizeof(float) * 8 * nr, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(recovered_idx, d_rec_idx, sizeof(int32_t) * nr, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(recovered_board, d_rec_board, sizeof(int32_t) * nr, cudaMemcpyDeviceToHost));
    }
    *n_out = out[0];
    return FID_OK;
}

extern "C" int fid_set_batch_marker_refinement(fid_detector* h, int enable) {
    if (!h || h->pend_count) return FID_ERR_INVALID_ARG;
    if (enable && (h->multi || h->aruco3.enable || h->marker_conf || h->inverted)) return FID_ERR_UNSUPPORTED;
    if (enable) {  // (a failed allocation leaves the option off; the next enable completes it)
        CK(cudaSetDevice(h->device));
        const size_t F = h->max_batch, M = F * h->max_markers;
        int rc;
#define A(expr)                  \
    if ((rc = (expr)) != FID_OK) return rc;
        for (int i = 0; i < h->n_slots; i++) {
            Slot& s = h->slot[i];
            if (!s.d_rej_n) A(dalloc(&s.d_rej_n, F));
            if (!s.d_rej) A(dalloc(&s.d_rej, F * h->max_sel * 8));
            if (!s.d_mr_nrec) A(dalloc(&s.d_mr_nrec, F));
            if (!s.d_mr_idx) A(dalloc(&s.d_mr_idx, M));
            if (!s.d_mr_board) A(dalloc(&s.d_mr_board, M));
            if (!s.h_rej_n) A(halloc(&s.h_rej_n, F));
            if (!s.h_rej) A(halloc(&s.h_rej, F * h->max_sel * 8));
            if (!s.h_mr_nrec) A(halloc(&s.h_mr_nrec, F));
            if (!s.h_mr_idx) A(halloc(&s.h_mr_idx, M));
            if (!s.h_mr_board) A(halloc(&s.h_mr_board, M));
        }
#undef A
        CK(cudaFuncSetAttribute(k_marker_refine, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)MREFINE_SMEM));
    }
    h->batch_refine = enable ? 1 : 0;
    return FID_OK;
}

extern "C" int fid_last_marker_refinement(fid_detector* h, int max_markers, int max_rejected, int* n_frames, int32_t* n_recovered, int32_t* recovered_idx,
                                          int32_t* recovered_board, int32_t* n_rejected, float* rejected) {
    if (!h || max_markers < 0 || max_rejected < 0) return FID_ERR_INVALID_ARG;
    if (!h->last_mr_valid) return FID_ERR_INVALID_ARG;
    const int nf = h->last_mr_frames;
    for (int f = 0; f < nf; f++)
        if (((recovered_idx || recovered_board) && h->last_mr_nrec[f] > max_markers) || (rejected && h->last_mr_nrej[f] > max_rejected)) return FID_ERR_CAPACITY;
    if (n_frames) *n_frames = nf;
    size_t oi = 0, oj = 0;
    for (int f = 0; f < nf; f++) {
        const int nr = h->last_mr_nrec[f], nj = h->last_mr_nrej[f];
        if (n_recovered) n_recovered[f] = nr;
        if (n_rejected) n_rejected[f] = nj;
        if (recovered_idx) memcpy(recovered_idx + (size_t)f * max_markers, h->last_mr_idx.data() + oi, sizeof(int32_t) * nr);
        if (recovered_board) memcpy(recovered_board + (size_t)f * max_markers, h->last_mr_board.data() + oi, sizeof(int32_t) * nr);
        if (rejected) memcpy(rejected + (size_t)f * max_rejected * 8, h->last_mr_rej.data() + oj * 8, sizeof(float) * 8 * nj);
        oi += nr;
        oj += nj;
    }
    return FID_OK;
}

// fid_set_diamonds (family < 0: no family, refused in multi-dictionary mode) and fid_set_family_diamonds
static int set_diamonds(fid_detector* h, const fid_diamond_params* params, int32_t family) {
    if (!h || !params || h->pend_count) return FID_ERR_INVALID_ARG;  // batches in flight read the layout
    const fid_diamond_params p = *params;
    if (family >= h->n_dicts) return FID_ERR_INVALID_ARG;
    if (p.enable && h->multi && family < 0) return FID_ERR_UNSUPPORTED;
    DiamondLayout L{};
    if (p.enable) {
        if (!std::isfinite(p.square_length) || !(p.marker_length > 0) || !(p.marker_length < p.square_length)) return FID_ERR_INVALID_ARG;
        if (p.min_markers < 0 || p.min_markers > 2) return FID_ERR_INVALID_ARG;  // cv2 asserts outside 0..2
        if (!diamond_layout(p.square_length, p.marker_length, p.min_markers, p.check_markers ? 1 : 0, &L)) return FID_ERR_INVALID_ARG;
        CK(cudaSetDevice(h->device));
        int rc;  // (a failed allocation leaves the option off; the next enable completes it)
        for (int i = 0; i < h->n_slots; i++) {
            Slot& s = h->slot[i];
            if (!s.d_dia_n && (rc = dalloc(&s.d_dia_n, (size_t)h->max_batch)) != FID_OK) return rc;
            if (!s.d_dia && (rc = dalloc(&s.d_dia, (size_t)h->max_batch * FID_MAX_DIAMONDS)) != FID_OK) return rc;
            if (!s.h_dia_n && (rc = halloc(&s.h_dia_n, (size_t)h->max_batch)) != FID_OK) return rc;
            if (!s.h_dia && (rc = halloc(&s.h_dia, (size_t)h->max_batch * FID_MAX_DIAMONDS)) != FID_OK) return rc;
        }
        if (!h->d_dia_io && (rc = dalloc(&h->d_dia_io, 2)) != FID_OK) return rc;
        if (!h->d_dia_list && (rc = dalloc(&h->d_dia_list, FID_MAX_DIAMONDS)) != FID_OK) return rc;
        if (!h->d_ch_masks) {  // the chessboard corners' cornerSubPix table, shared with the ChArUco boards
            std::vector<float> masks(FID_CHARUCO_MASK_FLOATS);
            charuco_subpix_masks(masks.data());
            if ((rc = dalloc(&h->d_ch_masks, masks.size())) != FID_OK) return rc;
            CK(cudaMemcpy(h->d_ch_masks, masks.data(), sizeof(float) * masks.size(), cudaMemcpyHostToDevice));
            CK(cudaFuncSetAttribute(k_charuco, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CHARUCO_SMEM));
        }
    }
    h->diamond = p;
    h->diamond.enable = p.enable ? 1 : 0;
    h->diamond_layout = L;
    h->diamond_fam = family < 0 ? 0 : family;
    h->diamond_bound = family >= 0;
    return FID_OK;
}

extern "C" int fid_set_diamonds(fid_detector* h, const fid_diamond_params* params) { return set_diamonds(h, params, -1); }

extern "C" int fid_set_family_diamonds(fid_detector* h, const fid_diamond_params* params, int32_t dict_index) {
    if (dict_index < 0) return FID_ERR_INVALID_ARG;
    return set_diamonds(h, params, dict_index);
}

extern "C" int fid_detect_diamonds(fid_detector* h, const uint8_t* bgr, int width, int height, size_t stride, int n, const int32_t* ids, const float* corners,
                                   const fid_camera* cam, int* n_diamonds, fid_diamond* out) {
    if (!h || !bgr || !n_diamonds || n < 0 || n > FID_MAX_MARKERS || (n > 0 && (!ids || !corners)) || (n >= 4 && !out) || !h->diamond.enable) return FID_ERR_INVALID_ARG;
    if (h->multi) return FID_ERR_UNSUPPORTED;  // the list carries no family: the batch calls serve this mode
    if (width < 16 || height < 16 || width > h->max_w || height > h->max_h || stride < (size_t)width * h->bpp) return FID_ERR_INVALID_ARG;
    if (h->pend_count) return FID_ERR_INVALID_ARG;  // slot 0 may belong to a batch in flight
    CK(cudaSetDevice(h->device));
    Slot& s = h->slot[0];
    CK(cudaMemcpy2DAsync(s.d_bgr, (size_t)width * h->bpp, bgr, stride, (size_t)width * h->bpp, height, cudaMemcpyHostToDevice, h->stream));
    if (n > 0) {
        CK(cudaMemcpyAsync(h->d_pose_ids, ids, sizeof(int32_t) * n, cudaMemcpyHostToDevice, h->stream));
        CK(cudaMemcpyAsync(h->d_pose_corners, corners, sizeof(float) * 8 * n, cudaMemcpyHostToDevice, h->stream));
    }
    CK(cudaMemcpyAsync(h->d_dia_io, &n, sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
    DiamondArgs a = diamond_args(h, s.d_bgr, (size_t)width * h->bpp, (size_t)width * h->bpp * height, width, height, cam);
    a.max_markers = FID_MAX_MARKERS;
    a.count = h->d_dia_io;
    a.ids = h->d_pose_ids;
    a.corners = h->d_pose_corners;
    a.n_out = h->d_dia_io + 1;
    a.out = h->d_dia_list;
    k_diamond<<<1, DIAMOND_THREADS, 0, h->stream>>>(a);
    CK(cudaGetLastError());
    int32_t nd = 0;
    CK(cudaMemcpyAsync(&nd, h->d_dia_io + 1, sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    if (nd > 0) CK(cudaMemcpy(out, h->d_dia_list, sizeof(fid_diamond) * nd, cudaMemcpyDeviceToHost));
    *n_diamonds = nd;
    return FID_OK;
}

extern "C" int fid_last_diamonds(fid_detector* h, int max_diamonds, int* n_frames, int32_t* counts, fid_diamond* out) {
    if (!h || max_diamonds < 0 || !h->last_dia_valid) return FID_ERR_INVALID_ARG;
    const int nf = h->last_dia_frames;
    if (out)
        for (int f = 0; f < nf; f++)
            if (h->last_dia_n[f] > max_diamonds) return FID_ERR_CAPACITY;
    if (n_frames) *n_frames = nf;
    size_t o = 0;
    for (int f = 0; f < nf; f++) {
        const int nd = h->last_dia_n[f];
        if (counts) counts[f] = nd;
        if (out) memcpy(out + (size_t)f * max_diamonds, h->last_dia.data() + o, sizeof(fid_diamond) * nd);
        o += nd;
    }
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

extern "C" int fid_debug_rejected(fid_detector* h, int max_rejected, int* n, float* rejected) {
    if (!h || !n || max_rejected < 0 || h->pend_count) return FID_ERR_INVALID_ARG;
    if (!h->detected) return FID_ERR_INVALID_ARG;  // slot 0's candidate lists were never written
    if (h->detected_multi) return FID_ERR_UNSUPPORTED;  // detectMarkersMultiDict's rejected list (DESIGN.md finding 15) is not modelled
    if (h->aruco3.enable) return FID_ERR_UNSUPPORTED;   // nor is the rejected list of useAruco3Detection (finding 16)
    if (h->inverted) return FID_ERR_UNSUPPORTED;        // nor the one of detectInvertedMarker (finding 18)
    CK(cudaSetDevice(h->device));
    int rc;
    if (!h->d_dbg_rej_n && (rc = dalloc(&h->d_dbg_rej_n, 1)) != FID_OK) return rc;
    if (!h->d_dbg_rej && (rc = dalloc(&h->d_dbg_rej, (size_t)h->max_sel * 8)) != FID_OK) return rc;
    Slot& s = h->slot[0];
    RejectedArgs a{};
    a.n_sel = s.d_nsel;
    a.cand_id = s.d_cand_id;
    a.fs = s.fs;
    a.max_raw = h->max_raw;
    a.max_sel = h->max_sel;
    a.n_rej = h->d_dbg_rej_n;
    a.rej = h->d_dbg_rej;
    k_rejected<<<1, FINISH_THREADS, 0, h->stream>>>(a);
    CK(cudaGetLastError());
    int32_t cnt = 0;
    CK(cudaMemcpyAsync(&cnt, h->d_dbg_rej_n, sizeof(cnt), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    *n = cnt;
    if (cnt > max_rejected) return FID_ERR_CAPACITY;
    if (cnt > 0 && rejected) CK(cudaMemcpy(rejected, h->d_dbg_rej, sizeof(float) * 8 * cnt, cudaMemcpyDeviceToHost));
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
