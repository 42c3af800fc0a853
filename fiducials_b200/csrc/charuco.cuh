// ChArUco boards: the chessboard corners of cv::aruco::CharucoBoard, found from markers that are already detected as
// cv::aruco::CharucoDetector::detectBoard(image, charucoCorners, charucoIds, markerCorners, markerIds) of OpenCV 4.13 finds them
// (objdetect/src/aruco/charuco_detector.cpp), and the board pose of CharucoBoard::matchImagePoints + cv::solvePnP(ITERATIVE).
//
//   layout      CharucoBoard(size, squareLength, markerLength, dict, ids): a marker in every white square (row-major, the legacy
//               pattern flips the colours of boards with an even row count), chessboard corner (x, y) at ((x + 1) s, (y + 1) s),
//               and per corner its nearest markers (centre distances within (0.01 s)^2 are ties) with each one's nearest corner.
//   position    with a camera (interpolateCornersCharucoApproxCalib): solvePnP over the matched marker corners (board_pnp.cuh),
//               then projectPoints of every corner, rounded to float32.  Without (interpolateCornersCharucoLocalHom): per nearest
//               marker, getPerspectiveTransform from its 2-D object corners to its first detection's corners (invalid when
//               |det| <= 1e-6) and perspectiveTransform of the corner; two positions are averaged, none gives (-1, -1).
//   window      getMaximumSubPixWindowSizes: int(min distance to the nearest markers' nearest detected corners - 2), in 1..10;
//               -1 (the detector's cornerRefinementWinSize) when no nearest marker is detected.
//   refinement  selectAndRefineChessboardCorners: corners whose rounded position lies in the image less 2 px on every side, in
//               ascending id; cornerSubPix on the position - 0.5 px, + 0.5 px after.
//   filters     filterCornersWithoutMinMarkers (minMarkers of the nearest markers detected), then with checkMarkers the board check
//               (CharucoDetectorImpl::checkBoard) that drops every corner when a marker contradicts the layout.
//   pose        matchImagePoints of the corners in output order and solve_board_pose; needs a camera, 4 corners and corners that are
//               not collinear (CharucoBoard::checkCharucoCornersCollinear).
//
// The float32 / float64 mix of each step is OpenCV's: getPerspectiveTransform forms -src.x * dst.x in float32, perspectiveTransform
// and the window distance work in double on float32 points, the mean of two positions and the board check work in float32.
#pragma once
#include <float.h>

#include "board_pnp.cuh"
#include "subpix.cuh"

namespace fid {

#define FID_CHARUCO_MAX_WIN 10  // getMaximumSubPixWindowSizes' upper bound
#define FID_CHARUCO_MASK_FLOATS 1770  // cornerSubPix masks of the windows 1..10, concatenated

// One board as the device reads it.  Marker tables hold n_markers rows, corner tables n_corners rows.
struct CharucoView {
    int n_markers, n_corners;
    int min_markers, check_markers;
    const int32_t* keys;         // board ids, sorted
    const int32_t* marker_of;    // board marker index of each sorted id
    const int32_t* ids;          // [n_markers] ids in board order
    const float* obj;            // [n_markers][4][3] marker corners (CharucoBoard::getObjPoints)
    const float* chess;          // [n_corners][3] chessboard corners (getChessboardCorners)
    const int32_t* near_n;       // [n_corners] number of nearest markers (1 or 2)
    const int32_t* near_idx;     // [n_corners][2] their board marker indices
    const int32_t* near_corner;  // [n_corners][2] the corner of each that is nearest to the chessboard corner
};

// ---- layout (host) ----------------------------------------------------------------------------------------------------------------
// The cornerSubPix weights of the windows 1..10, concatenated (FID_CHARUCO_MASK_FLOATS).  selectAndRefineChessboardCorners passes
// zeroZone = Size(), that is (0, 0), not (-1, -1): the centre weight of every window is 0, unlike the marker corners' table.
inline void charuco_subpix_masks(float* out) {
    for (int w = 1; w <= FID_CHARUCO_MAX_WIN; w++) {
        const int ww = 2 * w + 1;
        for (int i = 0; i < ww; i++) {  // as params_host.h's subpix_mask (host libm expf)
            const float y = (float)(i - w) / w;
            const float vy = expf(-y * y);
            for (int j = 0; j < ww; j++) {
                const float x = (float)(j - w) / w;
                out[i * ww + j] = (float)(vy * expf(-x * x));
            }
        }
        out[w * ww + w] = 0.f;
        out += ww * ww;
    }
}

// The counts of a board: markers floor(sx sy / 2), corners (sx - 1)(sy - 1).
inline int charuco_n_markers(int sx, int sy) { return sx * sy / 2; }
inline int charuco_n_corners(int sx, int sy) { return (sx - 1) * (sy - 1); }

// CharucoBoardImpl::createCharucoBoard + calcNearestMarkerCorners.  obj [n_markers][12], chess [n_corners][3], near_* [n_corners]
// ([2] for idx and corner).  Returns false if a corner has more than 2 nearest markers (no board of this shape has).
inline bool charuco_layout(int sx, int sy, float square, float marker, bool legacy, float* obj, float* chess, int32_t* near_n, int32_t* near_idx,
                           int32_t* near_corner) {
    const float diff = (square - marker) / 2;
    int m = 0;
    for (int y = 0; y < sy; y++)
        for (int x = 0; x < sx; x++) {
            if (legacy && (sy % 2 == 0)) {
                if ((y + 1) % 2 == x % 2) continue;
            } else if (y % 2 == x % 2) {
                continue;
            }
            float* o = obj + (size_t)m * 12;
            const float x0 = x * square + diff, y0 = y * square + diff;
            const float c[4][2] = {{x0, y0}, {x0 + marker, y0}, {x0 + marker, y0 + marker}, {x0, y0 + marker}};
            for (int k = 0; k < 4; k++) {
                o[3 * k] = c[k][0];
                o[3 * k + 1] = c[k][1];
                o[3 * k + 2] = 0.f;
            }
            m++;
        }
    const int nc = (sx - 1) * (sy - 1);
    for (int y = 0; y < sy - 1; y++)
        for (int x = 0; x < sx - 1; x++) {
            float* c = chess + (size_t)(y * (sx - 1) + x) * 3;
            c[0] = (x + 1) * square;
            c[1] = (y + 1) * square;
            c[2] = 0.f;
        }
    const double tie = (0.01 * square) * (0.01 * square);  // cv::pow(0.01 * squareLength, 2)
    for (int i = 0; i < nc; i++) {
        const float* cc = chess + (size_t)i * 3;
        int cnt = 0, idx[8];
        double min_d = -1;
        for (int j = 0; j < m; j++) {
            const float* o = obj + (size_t)j * 12;
            float cx = 0.f, cy = 0.f;
            for (int k = 0; k < 4; k++) {
                cx += o[3 * k];
                cy += o[3 * k + 1];
            }
            cx = (float)(cx / 4.);
            cy = (float)(cy / 4.);
            const float dx = cc[0] - cx, dy = cc[1] - cy;
            const double d = dx * dx + dy * dy;  // float, as Point3f
            if (j == 0 || fabs(d - min_d) < tie) {
                if (cnt == 8) return false;
                idx[cnt++] = j;
                min_d = d;
            } else if (d < min_d) {
                cnt = 0;
                idx[cnt++] = j;
                min_d = d;
            }
        }
        if (cnt > 2) return false;
        near_n[i] = cnt;
        for (int j = 0; j < 2; j++) {
            near_idx[2 * i + j] = j < cnt ? idx[j] : -1;
            near_corner[2 * i + j] = -1;
        }
        for (int j = 0; j < cnt; j++) {
            const float* o = obj + (size_t)idx[j] * 12;
            double best = -1;
            for (int k = 0; k < 4; k++) {
                const float dx = cc[0] - o[3 * k], dy = cc[1] - o[3 * k + 1];
                const double d = dx * dx + dy * dy;
                if (k == 0 || d < best) {
                    best = d;
                    near_corner[2 * i + j] = k;
                }
            }
        }
    }
    return true;
}

// ---- per-marker and per-corner arithmetic (host and device) ------------------------------------------------------------------------
// The first detection (in detection order) of id, or -1.
FID_HD int charuco_first_detection(int n_det, const int32_t* det_ids, int id) {
    for (int j = 0; j < n_det; j++)
        if (det_ids[j] == id) return j;
    return -1;
}

// cv::getPerspectiveTransform(src, dst) (DECOMP_LU) of 4 float32 point pairs; returns false where the LU finds the system singular
// (cv::solve then gives zeros).  M[8] = 1.
FID_HD bool charuco_perspective_transform(const float src[8], const float dst[8], double M[9]) {
    double a[8][8], b[8];
    for (int i = 0; i < 4; i++) {
        const float sx = src[2 * i], sy = src[2 * i + 1], dx = dst[2 * i], dy = dst[2 * i + 1];
        a[i][0] = a[i + 4][3] = sx;
        a[i][1] = a[i + 4][4] = sy;
        a[i][2] = a[i + 4][5] = 1;
        a[i][3] = a[i][4] = a[i][5] = a[i + 4][0] = a[i + 4][1] = a[i + 4][2] = 0;
        a[i][6] = -sx * dx;  // float32 products
        a[i][7] = -sy * dx;
        a[i + 4][6] = -sx * dy;
        a[i + 4][7] = -sy * dy;
        b[i] = dx;
        b[i + 4] = dy;
    }
    // hal::LU64f (LUImpl): partial pivoting, eps = 100 DBL_EPSILON
    for (int i = 0; i < 8; i++) {
        int k = i;
        for (int j = i + 1; j < 8; j++)
            if (fabs(a[j][i]) > fabs(a[k][i])) k = j;
        if (fabs(a[k][i]) < 2.220446049250313e-16 * 100) {
            for (int r = 0; r < 8; r++) M[r] = 0.0;
            M[8] = 1.0;
            return false;
        }
        if (k != i) {
            for (int j = i; j < 8; j++) {
                const double t = a[i][j];
                a[i][j] = a[k][j];
                a[k][j] = t;
            }
            const double t = b[i];
            b[i] = b[k];
            b[k] = t;
        }
        const double d = -1 / a[i][i];
        for (int j = i + 1; j < 8; j++) {
            const double alpha = a[j][i] * d;
            for (int c = i + 1; c < 8; c++) a[j][c] += alpha * a[i][c];
            b[j] += alpha * b[i];
        }
    }
    for (int i = 7; i >= 0; i--) {
        double s = b[i];
        for (int k = i + 1; k < 8; k++) s -= a[i][k] * b[k];
        b[i] = s / a[i][i];
    }
    for (int r = 0; r < 8; r++) M[r] = b[r];
    M[8] = 1.0;
    return true;
}

// cv::determinant of a 3x3 CV_64F matrix.
FID_HD double charuco_det3(const double m[9]) {
    return m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) + m[2] * (m[3] * m[7] - m[4] * m[6]);
}

// cv::perspectiveTransform of one float32 point (perspectiveTransform_32f).
FID_HD void charuco_apply(const double m[9], float x, float y, float out[2]) {
    const double X = x, Y = y;
    double w = X * m[6] + Y * m[7] + m[8];
    if (fabs(w) > 1.1920928955078125e-07) {
        w = 1. / w;
        out[0] = (float)((X * m[0] + Y * m[1] + m[2]) * w);
        out[1] = (float)((X * m[3] + Y * m[4] + m[5]) * w);
    } else {
        out[0] = out[1] = 0.f;
    }
}

// interpolateCornersCharucoLocalHom for corner i: xy = (-1, -1) when none of its nearest markers has a valid transform.
FID_HD void charuco_corner_local(const CharucoView& B, int i, int n_det, const int32_t* det_ids, const float* det_corners, float xy[2]) {
    float pos[2][2];
    int np = 0;
    for (int j = 0; j < B.near_n[i]; j++) {
        const int mk = B.near_idx[2 * i + j];
        const int d = charuco_first_detection(n_det, det_ids, B.ids[mk]);
        if (d < 0) continue;
        float src[8];
        for (int k = 0; k < 4; k++) {
            src[2 * k] = B.obj[(size_t)mk * 12 + 3 * k];
            src[2 * k + 1] = B.obj[(size_t)mk * 12 + 3 * k + 1];
        }
        double M[9];
        charuco_perspective_transform(src, det_corners + (size_t)d * 8, M);
        if (!(fabs(charuco_det3(M)) > 1e-6)) continue;
        charuco_apply(M, B.chess[3 * i], B.chess[3 * i + 1], pos[np]);
        np++;
    }
    if (np == 0) {
        xy[0] = xy[1] = -1.f;
    } else if (np == 1) {
        xy[0] = pos[0][0];
        xy[1] = pos[0][1];
    } else {  // (p0 + p1) / 2.: a float32 sum, halved in double
        xy[0] = (float)((double)(pos[0][0] + pos[1][0]) / 2.);
        xy[1] = (float)((double)(pos[0][1] + pos[1][1]) / 2.);
    }
}

// getMaximumSubPixWindowSizes for corner i at xy: 1..10, or -1 (the detector's window).
FID_HD int charuco_window(const CharucoView& B, int i, const float xy[2], int n_det, const int32_t* det_ids, const float* det_corners) {
    if (xy[0] == -1.f && xy[1] == -1.f) return -1;
    double min_d = -1;
    int counter = 0;
    for (int j = 0; j < B.near_n[i]; j++) {
        const int mk = B.near_idx[2 * i + j];
        const int d = charuco_first_detection(n_det, det_ids, B.ids[mk]);
        if (d < 0) continue;
        const int c = B.near_corner[2 * i + j];
        const float dx = det_corners[(size_t)d * 8 + 2 * c] - xy[0], dy = det_corners[(size_t)d * 8 + 2 * c + 1] - xy[1];
        const double dist = sqrt((double)dx * dx + (double)dy * dy);
        if (min_d == -1) min_d = dist;
        min_d = dist < min_d ? dist : min_d;
        counter++;
    }
    if (counter == 0) return -1;
    int w = (int)(min_d - 2);
    w = w < 1 ? 1 : w;
    return w > 10 ? 10 : w;
}

// Rect(2, 2, W - 4, H - 4).contains(pt): the float32 point is converted to Point (cvRound) first.
FID_HD bool charuco_inside(const float xy[2], int W, int H) {
    if (!(fabsf(xy[0]) < 2.0e9f) || !(fabsf(xy[1]) < 2.0e9f)) return false;
    const int x = (int)rint(xy[0]), y = (int)rint(xy[1]);
    return 2 <= x && x < 2 + (W - 4) && 2 <= y && y < 2 + (H - 4);
}

// cornerSubPix of one corner as selectAndRefineChessboardCorners runs it: on xy - 0.5 px, window win (1..10), + 0.5 px after.
// masks: the windows 1..10 concatenated; patch: (2 FID_CHARUCO_MAX_WIN + 3)^2 floats of scratch.
template <class Img>
FID_HD void charuco_refine(const Img& gray, int W, int H, float xy[2], int win, const float* masks, int max_iters, double eps_sq, float* patch) {
    int off = 0;
    for (int w = 1; w < win; w++) off += (2 * w + 1) * (2 * w + 1);
    float x = xy[0] - 0.5f, y = xy[1] - 0.5f;
    corner_subpix(gray, W, H, &x, &y, win, masks + off, max_iters, eps_sq, patch);
    xy[0] = x + 0.5f;
    xy[1] = y + 0.5f;
}

// filterCornersWithoutMinMarkers: how many of corner i's nearest markers were detected at all.
FID_HD int charuco_marker_count(const CharucoView& B, int i, int n_det, const int32_t* det_ids) {
    int cnt = 0;
    for (int j = 0; j < B.near_n[i]; j++) cnt += charuco_first_detection(n_det, det_ids, B.ids[B.near_idx[2 * i + j]]) >= 0;
    return cnt;
}

// CharucoDetectorImpl::checkBoard for one output corner (id ch at xy): false if the detected board markers contradict the layout
// there.  det_k[j] = the board marker index of detection j, or -1.
FID_HD bool charuco_check_corner(const CharucoView& B, int ch, const float xy[2], int n_det, const int32_t* det_ids, const int32_t* det_k, const float* det_corners) {
    float dx_max = 0.f, dy_min = FLT_MAX;
    const int n_near = B.near_n[ch];
    for (int j = 0; j < n_det; j++) {
        if (det_k[j] < 0) continue;
        const float* c = det_corners + (size_t)j * 8;
        const float mx = (c[0] + c[2] + c[4] + c[6]) / 4.f, my = (c[1] + c[3] + c[5] + c[7]) / 4.f;
        const float ex = mx - xy[0], ey = my - xy[1];
        const float dist = sqrtf(ex * ex + ey * ey);
        int which = -1;
        for (int q = 0; q < n_near && which < 0; q++)
            if (B.ids[B.near_idx[2 * ch + q]] == det_ids[j]) which = q;
        if (which >= 0) {
            const int nc = B.near_corner[2 * ch + which];
            const float nx = c[2 * nc], ny = c[2 * nc + 1];
            const float fx = nx - xy[0], fy = ny - xy[1];
            const float to_near = sqrtf(fx * fx + fy * fy);
            dx_max = dx_max > to_near ? dx_max : to_near;
            const int c1 = (nc + 1) % 4, c3 = (nc + 3) % 4;
            const float m1x = (c[2 * c1] + nx) * 0.5f, m1y = (c[2 * c1 + 1] + ny) * 0.5f;
            const float m2x = (c[2 * c3] + nx) * 0.5f, m2y = (c[2 * c3 + 1] + ny) * 0.5f;
            const float g1x = m1x - xy[0], g1y = m1y - xy[1], g2x = m2x - xy[0], g2y = m2y - xy[1];
            const float d1 = sqrtf(g1x * g1x + g1y * g1y), d2 = sqrtf(g2x * g2x + g2y * g2y);
            if ((d1 < d2 ? d1 : d2) < to_near) return false;
        } else {
            dy_min = dy_min < dist ? dy_min : dist;
        }
    }
    return !(dx_max > 0.f && dy_min < FLT_MAX && dx_max > dy_min);
}

// CharucoBoard::checkCharucoCornersCollinear over the ids of the output corners.
FID_HD bool charuco_collinear(const CharucoView& B, int n, const int32_t* ids) {
    if (n <= 2) return true;
    const double p0[3] = {B.chess[3 * ids[0]], B.chess[3 * ids[0] + 1], 1}, p1[3] = {B.chess[3 * ids[1]], B.chess[3 * ids[1] + 1], 1};
    double L[3] = {p0[1] * p1[2] - p0[2] * p1[1], p0[2] * p1[0] - p0[0] * p1[2], p0[0] * p1[1] - p0[1] * p1[0]};
    const double div = sqrt(L[0] * L[0] + L[1] * L[1]);
    for (int k = 0; k < 3; k++) L[k] /= div;
    for (int i = 2; i < n; i++) {
        const double dot = B.chess[3 * ids[i]] * L[0] + B.chess[3 * ids[i] + 1] * L[1] + 1 * L[2];
        if (fabs(dot) > 1e-6) return false;
    }
    return true;
}

// Chessboard corner i projected through the approximate pose (cv::projectPoints, rounded to float32).
FID_HD void charuco_project(const CharucoView& B, int i, const double R[9], const double p[6], const Camera& cam, float xy[2]) {
    double uv[2];
    project_point(B.chess[3 * i], B.chess[3 * i + 1], B.chess[3 * i + 2], R, nullptr, p, cam, uv, nullptr);
    xy[0] = (float)uv[0];
    xy[1] = (float)uv[1];
}

}  // namespace fid
