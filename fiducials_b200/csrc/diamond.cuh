// ChArUco diamonds: cv::aruco::CharucoDetector::detectDiamonds(image, diamondCorners, diamondIds, markerCorners, markerIds) of OpenCV
// 4.13 (objdetect/src/aruco/charuco_detector.cpp) for markers that are already detected, restated for host and device.  A diamond
// is a 3x3 chessboard with four markers around the centre square, named by the four marker ids.
//
//   layout      CharucoBoard((3, 3), squareLength, markerLength): markers top, left, right, bottom (board order), chessboard
//               corners (1, 1), (2, 1), (1, 2), (2, 2) squares (charuco_layout).
//   loop        nothing with fewer than 4 markers.  Each marker i in list order that is not assigned yet: minRepDistance =
//               sqrtf(sum of the squared side lengths) * 1.302455f (float32; the root of the sum of squares, not the perimeter);
//               the candidates are the other unassigned markers in list order, and the loop ends (break) when there are fewer than
//               3.  The temporary board has the ids {id_i, id_i + 2, id_i + 3, id_i + 4}, so marker i is its top marker in its own
//               corner order.  refineDetectedMarkers(grey, board, [marker i], candidates) with RefineParameters(minRepDistance, -1,
//               false) and no camera: the homography of marker i's corners (board_homography) predicts the left, right and bottom
//               markers (refine_transform), each takes the nearest candidate not taken yet with rotation 0 only and no bit check
//               (refine_match).  When all three are recovered the four markers are assigned and the diamond's ids are {id_i, the
//               ids of the markers recovered for left, right, bottom}.
//   corners     the recovered markers' corners get cornerSubPix under CORNER_REFINE_SUBPIX (refine_subpix_corner), written back
//               into the marker list (see diamond_assign); then detectBoard on the temporary board with the four markers and the temporary ids: the detector's camera if one is set
//               (solvePnP over the 16 marker corners, projectPoints), local homographies otherwise; border, minMarkers, window and
//               cornerSubPix as for any ChArUco board, and checkMarkers' board check.  The diamond is kept when all 4 corners
//               survive, its corners reordered 0, 1, 3, 2.  cv2 indexes past the end of a list of 1 to 3 corners (a diamond at the
//               image border); such a diamond is dropped here (DESIGN.md finding 13).
//   pose        cv::solvePnP(ITERATIVE) of the 4 corners on getSingleMarkerObjectPoints(squareLength): solve_marker_pose with the
//               square length as the marker length.
//
// Every diamond is found in the order of the loop.
#pragma once
#include "charuco.cuh"
#include "marker_refine.cuh"
#include "pnp.cuh"

namespace fid {

// The temporary 3x3 board, shared by every diamond of one geometry.  rows: the board row of each sorted id -- the temporary ids
// ascend in board order, so it is the identity.
struct DiamondLayout {
    float obj[4 * 12];   // [4][4][3] marker corners, board order
    float chess[4 * 3];  // [4][3] chessboard corners
    int32_t near_n[4], near_idx[8], near_corner[8];
    int32_t rows[4];
    int32_t min_markers, check_markers;
    float square_length;
};

inline bool diamond_layout(float square, float marker, int min_markers, int check_markers, DiamondLayout* D) {
    for (int k = 0; k < 4; k++) D->rows[k] = k;
    D->min_markers = min_markers;
    D->check_markers = check_markers;
    D->square_length = square;
    return charuco_layout(3, 3, square, marker, false, D->obj, D->chess, D->near_n, D->near_idx, D->near_corner);
}

// The temporary board of a diamond whose four markers (in board order) carry the temporary ids tmp[4].
FID_HD CharucoView diamond_view(const DiamondLayout& D, const int32_t tmp[4]) {
    return CharucoView{4, 4, D.min_markers, D.check_markers, tmp, D.rows, tmp, D.obj, D.chess, D.near_n, D.near_idx, D.near_corner};
}

FID_HD void diamond_tmp_ids(int id, int32_t tmp[4]) {
    tmp[0] = id;
    for (int k = 1; k < 4; k++) tmp[k] = id + 1 + k;
}

// minRepDistance of marker corners c (float32 as cv2: Point2f differences, the sum of squares, sqrt of a float).
FID_HD float diamond_min_rep(const float c[8]) {
    float p = 0.f;
    for (int k = 0; k < 4; k++) {
        const int k1 = (k + 1) & 3;
        const float ex = c[2 * k] - c[2 * k1], ey = c[2 * k + 1] - c[2 * k1 + 1];
        p += ex * ex + ey * ey;
    }
    return sqrtf(p) * 1.302455f;
}

// refineDetectedMarkers' prediction with marker corners c as the top marker: the left, right and bottom markers, pred [3][8].  It
// depends on marker i alone, so it can be computed for every marker before the loop.  false where findHomography fails (nothing
// is recovered then).  Lanes as board_homography: one warp on the device.
FID_HD bool diamond_predict(const DiamondLayout& D, const float c[8], float pred[24]) {
    double Hm[9];
    if (!board_homography(4, [&](int i, float s[2], float d[2]) {
            s[0] = D.obj[3 * i];
            s[1] = D.obj[3 * i + 1];
            d[0] = c[2 * i];
            d[1] = c[2 * i + 1];
        }, Hm))
        return false;
    for (int r = 1; r < 4; r++) refine_transform(D.obj, r, Hm, pred + 8 * (r - 1));
    return true;
}

// Step "loop" over n markers whose corners wc [n][8] are a working copy of the list: under CORNER_REFINE_SUBPIX cv2 writes the
// cornerSubPix of every recovered marker back into the caller's markerCorners at once, whether or not a diamond follows (DESIGN.md
// finding 13), and every later step reads the list so changed.  pred [n][3][8] / pred_ok [n] are diamond_predict of the original
// corners; a marker whose corners changed (dirty [n]) is predicted again.  Output: the markers of every diamond found, dia [.][4]
// (the top marker, then the markers recovered for left, right and bottom), in order.  taken [n] is scratch: the assigned markers,
// and during one refineDetectedMarkers call also marker i and the candidates it took.  masks: the marker corners' cornerSubPix
// table (windows 1..5).  Returns the number of diamonds.  The lanes split each candidate screen (refine_match) and the four corners
// of a recovered marker; lane 0 writes the flags.
template <class Lanes, class Img>
FID_HD int diamond_assign(const Lanes& L, const Img& gray, int W, int H, const DevParams& P, const float* masks, const DiamondLayout& D, int n, float* wc, const float* pred,
                          const uint8_t* pred_ok, uint8_t* dirty, uint8_t* taken, int32_t* dia) {
    if (n < 4) return 0;
    for (int j = L.lane(); j < n; j += L.count()) taken[j] = dirty[j] = 0;
    L.sync();
    int nd = 0;
    for (int i = 0; i < n; i++) {
        if (taken[i]) continue;
        int free = 0;
        for (int j0 = 0; j0 < n; j0 += L.count()) {
            const int j = j0 + L.lane();
            free += fid_popc(L.ballot(j < n && j != i && !taken[j]));
        }
        if (free < 3) break;
        float pr[24];
        const float* pp = pred + (size_t)24 * i;
        if (dirty[i]) {
            if (!diamond_predict(D, wc + (size_t)8 * i, pr)) continue;
            pp = pr;
        } else if (!pred_ok[i]) {
            continue;
        }
        const MarkerRefineParams rp{diamond_min_rep(wc + (size_t)8 * i), -1.f, 0};
        if (L.lane() == 0) taken[i] = 1;
        L.sync();
        int got[3], k = 0;
        for (int r = 0; r < 3; r++) {  // after a miss the other positions still take candidates, and cornerSubPix changes them
            float q[8];
            const int j = refine_match(L, gray, W, H, P, nullptr, rp, -1, pp + 8 * r, n, wc, taken, nullptr, nullptr, q);
            if (j < 0) continue;
            got[k++] = j;
            if (P.corner_refine == 1) {
                for (int c = L.lane(); c < 4; c += L.count()) {
                    float xy[2], patch[(2 * FID_SUBPIX_MAX_WIN + 3) * (2 * FID_SUBPIX_MAX_WIN + 3)];
                    refine_subpix_corner(gray, W, H, P, masks, q, c, xy, patch);
                    wc[(size_t)8 * j + 2 * c] = xy[0];
                    wc[(size_t)8 * j + 2 * c + 1] = xy[1];
                }
                if (L.lane() == 0) dirty[j] = 1;
            }
            if (L.lane() == 0) taken[j] = 1;
            L.sync();
        }
        if (L.lane() == 0) {
            if (k == 3) {
                dia[4 * nd] = i;
                for (int m = 0; m < 3; m++) dia[4 * nd + 1 + m] = got[m];
            } else {
                taken[i] = 0;
                for (int m = 0; m < k; m++) taken[got[m]] = 0;
            }
        }
        L.sync();
        nd += k == 3;
    }
    return nd;
}

// Step "corners" for chessboard corner c of a diamond whose markers (board order, after cornerSubPix) are det [4][8]: position
// (through the approximate pose R, p with a camera), border and minMarkers filters, window and cornerSubPix.  false where the
// corner is dropped.  masks: charuco_subpix_masks; patch: (2 FID_CHARUCO_MAX_WIN + 3)^2 floats of scratch.
template <class Img>
FID_HD bool diamond_corner(const CharucoView& B, int c, bool has_cam, const double R[9], const double p[6], const Camera& cam, const Img& gray, int W, int H,
                           const float* det, const float* masks, int win_default, int max_iters, double eps_sq, float* patch, float xy[2]) {
    if (has_cam) charuco_project(B, c, R, p, cam, xy);
    else charuco_corner_local(B, c, 4, B.ids, det, xy);
    if (!charuco_inside(xy, W, H) || charuco_marker_count(B, c, 4, B.ids) < B.min_markers) return false;
    const int win = charuco_window(B, c, xy, 4, B.ids, det);
    charuco_refine(gray, W, H, xy, win < 0 ? win_default : win, masks, max_iters, eps_sq, patch);
    return true;
}

// The diamond's output position of chessboard corner c (0, 1, 3, 2).
FID_HD int diamond_slot(int c) { return c < 2 ? c : 5 - c; }

}  // namespace fid
