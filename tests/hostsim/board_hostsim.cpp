// CPU harness for fiducials_b200/csrc/board_pnp.cuh (one pose per marker board).  TEST INFRASTRUCTURE ONLY.
// Compiled with g++ by tests/test_hostsim_board.py into a shared object of its own in a temporary directory, from the same header
// the CUDA kernel k_board_pose is built from; it is not linked into libfiducials_b200.so.
#include <algorithm>
#include <vector>

#include "../../fiducials_b200/csrc/board_pnp.cuh"

using namespace fid;

namespace {

// The sorted (id, marker index) table fid_set_boards builds.
void board_table(int n_board, const int32_t* board_ids, std::vector<int32_t>& keys, std::vector<int32_t>& marker_of) {
    std::vector<int> ord(n_board);
    for (int i = 0; i < n_board; i++) ord[i] = i;
    std::sort(ord.begin(), ord.end(), [&](int a, int b) { return board_ids[a] < board_ids[b]; });
    keys.resize(n_board);
    marker_of.resize(n_board);
    for (int i = 0; i < n_board; i++) {
        keys[i] = board_ids[ord[i]];
        marker_of[i] = ord[i];
    }
}

}  // namespace

extern "C" {

// Board::matchImagePoints: obj_out [4 n][3], img_out [4 n][2] (capacity 4 n_det points); returns the matched marker count.
int hs_board_match(int n_det, const int32_t* det_ids, const float* det_corners, int n_board, const int32_t* board_ids, const float* board_obj, float* obj_out,
                   float* img_out) {
    std::vector<int32_t> keys, marker_of;
    board_table(n_board, board_ids, keys, marker_of);
    return board_match(n_det, det_ids, det_corners, n_board, keys.data(), marker_of.data(), board_obj, obj_out, img_out);
}

// findHomography(src, dst, 0) of n point pairs (given in double, converted to float32 as findHomography does); returns 0 if none.
int hs_homography(int n, const double* src, const double* dst, double* H) {
    return board_homography(n, [&](int i, float s[2], float d[2]) {
        s[0] = (float)src[2 * i];
        s[1] = (float)src[2 * i + 1];
        d[0] = (float)dst[2 * i];
        d[1] = (float)dst[2 * i + 1];
    }, H) ? 1 : 0;
}

// Match + solve for one board.  out: 20 doubles (status n_markers n_points rvec[3] tvec[3] quat[4] image_error lm_iters, pad)
void hs_board_pose(int n_det, const int32_t* det_ids, const float* det_corners, int n_board, const int32_t* board_ids, const float* board_obj, const double* K,
                   const double* D, double* out) {
    Camera cam = {K[0], K[4], K[2], K[5], D[0], D[1], D[2], D[3], D[4]};
    std::vector<float> obj((size_t)n_det * 12 + 1), img((size_t)n_det * 8 + 1);
    const int m = hs_board_match(n_det, det_ids, det_corners, n_board, board_ids, board_obj, obj.data(), img.data());
    std::vector<double> mn((size_t)m * 8 + 1);
    BoardPoseOut po;
    solve_board_pose(4 * m, obj.data(), img.data(), mn.data(), cam, &po);
    out[0] = po.status;
    out[1] = m;
    out[2] = po.n_points;
    for (int k = 0; k < 3; k++) {
        out[3 + k] = po.rvec[k];
        out[6 + k] = po.tvec[k];
    }
    for (int k = 0; k < 4; k++) out[9 + k] = po.quat[k];
    out[13] = po.image_error;
    out[14] = po.lm_iters;
}

}  // extern "C"
