// CPU harness for fiducials_b200/csrc/charuco.cuh (ChArUco corners and pose).  TEST INFRASTRUCTURE ONLY.
// Compiled with g++ by tests/test_hostsim_charuco.py into a shared object of its own in a temporary directory, from the same header
// the CUDA kernel k_charuco is built from; it is not linked into libfiducials_b200.so.  hs_charuco_detect runs the steps of
// k_charuco one after the other.
#include <algorithm>
#include <vector>

#include "../../fiducials_b200/csrc/charuco.cuh"

using namespace fid;

namespace {

struct HostBoard {
    int sx, sy, nm, nc;
    std::vector<int32_t> ids, keys, marker_of, near_n, near_idx, near_corner;
    std::vector<float> obj, chess;
    CharucoView view(int min_markers, int check_markers) const {
        return CharucoView{nm, nc, min_markers, check_markers, keys.data(), marker_of.data(), ids.data(), obj.data(), chess.data(), near_n.data(), near_idx.data(),
                           near_corner.data()};
    }
};

bool make_board(int sx, int sy, float square, float marker, int legacy, const int32_t* ids, HostBoard* b) {
    b->sx = sx;
    b->sy = sy;
    b->nm = charuco_n_markers(sx, sy);
    b->nc = charuco_n_corners(sx, sy);
    b->obj.resize((size_t)b->nm * 12 + 1);
    b->chess.resize((size_t)b->nc * 3 + 1);
    b->near_n.resize(b->nc + 1);
    b->near_idx.resize(2 * b->nc + 1);
    b->near_corner.resize(2 * b->nc + 1);
    if (!charuco_layout(sx, sy, square, marker, legacy != 0, b->obj.data(), b->chess.data(), b->near_n.data(), b->near_idx.data(), b->near_corner.data())) return false;
    b->ids.resize(b->nm);
    for (int i = 0; i < b->nm; i++) b->ids[i] = ids ? ids[i] : i;
    std::vector<int> ord(b->nm);
    for (int i = 0; i < b->nm; i++) ord[i] = i;
    std::sort(ord.begin(), ord.end(), [&](int x, int y) { return b->ids[x] < b->ids[y]; });
    for (int i = 0; i < b->nm; i++) {
        b->keys.push_back(b->ids[ord[i]]);
        b->marker_of.push_back(ord[i]);
    }
    return true;
}

std::vector<float> masks_1_10() {
    std::vector<float> masks(FID_CHARUCO_MASK_FLOATS);
    charuco_subpix_masks(masks.data());
    return masks;
}

}  // namespace

extern "C" {

// The layout: obj [n_markers][12], chess [n_corners][3], near_n [n_corners], near_idx / near_corner [n_corners][2].  Returns 1.
int hs_charuco_layout(int sx, int sy, float square, float marker, int legacy, float* obj, float* chess, int32_t* near_n, int32_t* near_idx, int32_t* near_corner) {
    return charuco_layout(sx, sy, square, marker, legacy != 0, obj, chess, near_n, near_idx, near_corner) ? 1 : 0;
}

// cornerSubPix of n points with window win (1..10) from the ChArUco mask table (zeroZone (0, 0)).
void hs_charuco_subpix(const uint8_t* gray, int W, int H, float* xy, int n, int win, int max_iters, double eps) {
    const std::vector<float> masks = masks_1_10();
    int off = 0;
    for (int w = 1; w < win; w++) off += (2 * w + 1) * (2 * w + 1);
    const GrayPlane img{gray, (size_t)W};
    std::vector<float> patch((2 * FID_CHARUCO_MAX_WIN + 3) * (2 * FID_CHARUCO_MAX_WIN + 3));
    for (int i = 0; i < n; i++) corner_subpix(img, W, H, &xy[2 * i], &xy[2 * i + 1], win, masks.data() + off, max_iters, eps * eps, patch.data());
}

// detectBoard with given markers (+ the pose).  K / D may be NULL (no camera).  refine: cornerRefinementWinSize, MaxIterations,
// MinAccuracy.  out_ids [n_corners], out_xy [n_corners][2], rec[16]: n status rvec[3] tvec[3] quat[4] image_error n_markers_matched.
// Returns the number of corners, or -1 for an invalid layout.
int hs_charuco_detect(int sx, int sy, float square, float marker, int legacy, const int32_t* board_ids, int min_markers, int check_markers, const uint8_t* gray,
                      int W, int H, int n_det, const int32_t* det_ids, const float* det_corners, const double* K, const double* D, int refine_win,
                      int refine_max_iter, double refine_min_acc, int32_t* out_ids, float* out_xy, double* rec) {
    HostBoard hb;
    if (!make_board(sx, sy, square, marker, legacy, board_ids, &hb)) return -1;
    const CharucoView B = hb.view(min_markers, check_markers);
    const std::vector<float> masks = masks_1_10();
    const GrayPlane img{gray, (size_t)W};
    std::vector<int32_t> det_k(n_det + 1);
    for (int j = 0; j < n_det; j++) {
        const int k = board_find(B.keys, B.n_markers, det_ids[j]);
        det_k[j] = k < 0 ? -1 : B.marker_of[k];
    }
    Camera cam{};
    if (K) cam = Camera{K[0], K[4], K[2], K[5], D[0], D[1], D[2], D[3], D[4]};
    // 1. positions
    std::vector<float> xy((size_t)2 * B.n_corners + 2);
    bool any = true;
    int m = 0;
    if (K) {
        std::vector<float> obj((size_t)n_det * 12 + 1), ip((size_t)n_det * 8 + 1);
        m = board_match(n_det, det_ids, det_corners, B.n_markers, B.keys, B.marker_of, B.obj, obj.data(), ip.data());
        any = m > 0;
        if (any) {
            std::vector<double> mn((size_t)m * 8 + 1);
            BoardPoseOut po;
            solve_board_pose(4 * m, obj.data(), ip.data(), mn.data(), cam, &po);
            double p[6] = {po.rvec[0], po.rvec[1], po.rvec[2], po.tvec[0], po.tvec[1], po.tvec[2]}, R[9];
            rodrigues_v2m(p, R, nullptr);
            for (int i = 0; i < B.n_corners; i++) charuco_project(B, i, R, p, cam, &xy[2 * i]);
        }
    } else {
        for (int i = 0; i < B.n_corners; i++) charuco_corner_local(B, i, n_det, det_ids, det_corners, &xy[2 * i]);
    }
    // 2. window, border, minMarkers, refinement; compaction in ascending id
    int n = 0;
    std::vector<float> patch((2 * FID_CHARUCO_MAX_WIN + 3) * (2 * FID_CHARUCO_MAX_WIN + 3));
    for (int i = 0; any && i < B.n_corners; i++) {
        float* c = &xy[2 * i];
        int win = charuco_window(B, i, c, n_det, det_ids, det_corners);
        if (!charuco_inside(c, W, H) || charuco_marker_count(B, i, n_det, det_ids) < B.min_markers) continue;
        charuco_refine(img, W, H, c, win < 0 ? refine_win : win, masks.data(), refine_max_iter, refine_min_acc * refine_min_acc, patch.data());
        out_ids[n] = i;
        out_xy[2 * n] = c[0];
        out_xy[2 * n + 1] = c[1];
        n++;
    }
    for (int k = 0; k < 16; k++) rec[k] = 0.0;
    rec[15] = m;
    // 3. checkBoard
    if (B.check_markers)
        for (int q = 0; q < n; q++)
            if (!charuco_check_corner(B, out_ids[q], &out_xy[2 * q], n_det, det_ids, det_k.data(), det_corners)) {
                rec[0] = 0;
                rec[1] = -3;
                return 0;
            }
    rec[0] = n;
    // 4. pose
    if (!K || n < 4) return n;
    if (charuco_collinear(B, n, out_ids)) {
        rec[1] = -2;
        return n;
    }
    std::vector<float> obj((size_t)n * 3);
    std::vector<double> mn((size_t)n * 2);
    for (int q = 0; q < n; q++)
        for (int k = 0; k < 3; k++) obj[3 * q + k] = B.chess[3 * out_ids[q] + k];
    BoardPoseOut po;
    solve_board_pose(n, obj.data(), out_xy, mn.data(), cam, &po);
    rec[1] = po.status;
    for (int k = 0; k < 3; k++) {
        rec[2 + k] = po.rvec[k];
        rec[5 + k] = po.tvec[k];
    }
    for (int k = 0; k < 4; k++) rec[8 + k] = po.quat[k];
    rec[12] = po.image_error;
    return n;
}

}  // extern "C"
