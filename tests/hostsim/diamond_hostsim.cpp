// CPU harness for fiducials_b200/csrc/diamond.cuh (ChArUco diamonds).  TEST INFRASTRUCTURE ONLY.
// Compiled with g++ by tests/test_hostsim_diamond.py into a shared object of its own in a temporary directory, from the same header
// the CUDA kernel k_diamond is built from; it is not linked into libfiducials_b200.so.  hs_diamonds runs the steps of k_diamond one
// after the other, with one lane.
#include <algorithm>
#include <vector>

#include "../../fiducials_b200/csrc/diamond.cuh"
#include "../../fiducials_b200/csrc/params_host.h"

using namespace fid;

extern "C" {

// detectDiamonds for n markers (ids [n], corners [n][8]) of a gray frame, with the detector parameters given (dictionary, corner
// method, cornerRefinementWinSize / MaxIterations / MinAccuracy, relativeCornerRefinmentWinSize).  K / D may be NULL.  Outputs per
// diamond, in order: out_ids [.][4], out_corners [.][8], out_pose [.][16] = status rvec[3] tvec[3] quat[4] image_error object_error
// area lm_iters.  out_wc [n][8] (may be NULL): the marker corners after the loop, as cv2 leaves markerCorners.  Returns the number of
// diamonds, or -1 for an invalid layout.
int hs_diamonds(const uint8_t* gray, int W, int H, int dictionary, int corner_method, int refine_win, int refine_max_iter, double refine_min_acc, double rel_refine_win,
                float square, float marker, int min_markers, int check_markers, int n, const int32_t* ids, const float* corners, const double* K, const double* D,
                int32_t* out_ids, float* out_corners, double* out_pose, float* out_wc) {
    fid_params fp;
    default_params(&fp);
    fp.dictionary = dictionary;
    fp.cornerRefinementMethod = corner_method;
    fp.cornerRefinementWinSize = refine_win;
    fp.cornerRefinementMaxIterations = refine_max_iter;
    fp.cornerRefinementMinAccuracy = refine_min_acc;
    fp.relativeCornerRefinmentWinSize = rel_refine_win;
    DevParams P;
    if (make_dev_params(fp, &P) != FID_OK) return -2;
    DiamondLayout DL;
    if (!diamond_layout(square, marker, min_markers, check_markers, &DL)) return -1;
    std::vector<float> masks;
    for (int w = 1; w <= 5; w++) {
        std::vector<float> m((2 * w + 1) * (2 * w + 1));
        subpix_mask(w, m.data());
        masks.insert(masks.end(), m.begin(), m.end());
    }
    std::vector<float> ch_masks(FID_CHARUCO_MASK_FLOATS);
    charuco_subpix_masks(ch_masks.data());
    Camera cam{};
    if (K) cam = Camera{K[0], K[4], K[2], K[5], D[0], D[1], D[2], D[3], D[4]};
    const GrayPlane img{gray, (size_t)W};
    const SerialLanes L;
    // 1. predictions, marker by marker
    std::vector<float> pred((size_t)24 * n + 1), wc(corners, corners + (size_t)8 * n);
    std::vector<uint8_t> ok(n + 1), taken(n + 1), dirty(n + 1);
    for (int i = 0; i < n; i++) ok[i] = diamond_predict(DL, corners + (size_t)8 * i, pred.data() + (size_t)24 * i);
    // 2. the loop, on a working copy of the corners
    std::vector<int32_t> dia((size_t)4 * (n / 4 + 1));
    const int nd = diamond_assign(L, img, W, H, P, masks.data(), DL, n, wc.data(), pred.data(), ok.data(), dirty.data(), taken.data(), dia.data());
    if (out_wc) std::copy(wc.begin(), wc.end(), out_wc);
    // 3. per diamond: the chessboard corners, the pose
    const int win_default = std::max(1, std::min(FID_CHARUCO_MAX_WIN, refine_win));
    const int max_iters = std::max(1, std::min(100, refine_max_iter));
    const double eps = std::max(refine_min_acc, 0.0);
    std::vector<float> patch((2 * FID_CHARUCO_MAX_WIN + 3) * (2 * FID_CHARUCO_MAX_WIN + 3));
    int q = 0;
    for (int k = 0; k < nd; k++) {
        const int32_t* m = dia.data() + 4 * k;
        float det[32];
        for (int r = 0; r < 4; r++)
            for (int c = 0; c < 8; c++) det[8 * r + c] = wc[(size_t)8 * m[r] + c];
        int32_t tmp[4];
        diamond_tmp_ids(ids[m[0]], tmp);
        const CharucoView B = diamond_view(DL, tmp);
        double R[9], p[6];
        if (K) {
            double mn[32];
            BoardPoseOut po;
            solve_board_pose(16, DL.obj, det, mn, cam, &po);
            for (int j = 0; j < 3; j++) {
                p[j] = po.rvec[j];
                p[3 + j] = po.tvec[j];
            }
            rodrigues_v2m(p, R, nullptr);
        }
        float xy[8];
        bool keep = true;
        for (int c = 0; c < 4 && keep; c++)
            keep = diamond_corner(B, c, K != nullptr, R, p, cam, img, W, H, det, ch_masks.data(), win_default, max_iters, eps * eps, patch.data(), xy + 2 * c);
        if (keep && DL.check_markers)
            for (int c = 0; c < 4 && keep; c++) keep = charuco_check_corner(B, c, xy + 2 * c, 4, tmp, DL.rows, det);
        if (!keep) continue;
        for (int r = 0; r < 4; r++) out_ids[4 * q + r] = ids[m[r]];
        for (int c = 0; c < 4; c++) {
            out_corners[8 * q + 2 * diamond_slot(c)] = xy[2 * c];
            out_corners[8 * q + 2 * diamond_slot(c) + 1] = xy[2 * c + 1];
        }
        double* o = out_pose + 16 * q;
        for (int j = 0; j < 16; j++) o[j] = 0.0;
        if (K) {
            PoseOut po;
            solve_marker_pose(out_corners + 8 * q, cam, square, (double)square, &po);
            o[0] = 1;
            for (int j = 0; j < 3; j++) {
                o[1 + j] = po.rvec[j];
                o[4 + j] = po.tvec[j];
            }
            for (int j = 0; j < 4; j++) o[7 + j] = po.quat[j];
            o[11] = po.image_error;
            o[12] = po.object_error;
            o[13] = po.area;
            o[14] = po.lm_iters;
        }
        q++;
    }
    return q;
}

}  // extern "C"
