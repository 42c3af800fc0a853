// Recovery of board markers that detection missed: cv::aruco::ArucoDetector::refineDetectedMarkers(image, board, detectedCorners,
// detectedIds, rejectedCorners, K, D, recoveredIdxs) of OpenCV 4.13 with RefineParameters (minRepDistance, errorCorrectionRate,
// checkAllOrders), restated for host and device.
//
//   prediction  with a camera: Board::matchImagePoints over the detections (detection order, repeats twice) and solvePnP
//               (board_pnp.cuh, solve_board_pose); nothing when no board marker is detected or where solvePnP raises (status -1).
//               Every board marker whose id is not among the detections, in board order, is projected with K and D (float32).
//               Without one: every board point must have the z of the first (cv2 asserts), findHomography(obj.xy -> corners)
//               over the four corners of the first detection of every detected board marker, in board order (board_homography),
//               then perspectiveTransform of every undetected marker (charuco_apply).
//   matching    greedy, in the order of the undetected markers, over the rejected candidates not taken yet.  The distance of a
//               corner order is the largest squared corner distance, in float32.  A rotation is kept when its distance is below the
//               best distance accepted so far for this marker, which starts at minRepDistance^2 + 1 (float32): with checkAllOrders
//               the LAST rotation below it wins, not the smallest.  With errorCorrectionRate >= 0 the rotated quad's inner bits
//               (extract_bits, identify.cuh) must differ from rotation 0 of the marker's code in fewer than
//               int(maxCorrectionBits * errorCorrectionRate) bits -- strictly fewer, so errorCorrectionRate 0 recovers nothing; there is
//               no border check.  A candidate that passes becomes the best so far; the best is taken.
//   corners     with CORNER_REFINE_SUBPIX the recovered corners get cornerSubPix with the detector's window rule
//               (min(round(relativeCornerRefinmentWinSize * module), cornerRefinementWinSize)) and zeroZone (-1, -1): the marker
//               corners' mask table.  NONE and CONTOUR leave them as matched.
//
// Several boards are consecutive calls: each sees the detections and the rejected list the previous call left.
#pragma once
#include "board_pnp.cuh"
#include "charuco.cuh"
#include "identify.cuh"
#include "subpix.cuh"

namespace fid {

struct MarkerRefineParams {
    float min_rep_distance;       // px, > 0
    float error_correction_rate;  // < 0: no bit check
    int check_all_orders;
};

// One board as refinement reads it: n markers, their ids sorted (keys) with each one's board row (marker_of), and the object points
// [n][4][3] in board order.
struct RefineBoardView {
    int n;
    const int32_t* keys;
    const int32_t* marker_of;
    const float* obj;
};

// closestCandidateDistance's start value: minRepDistance^2 + 1, in float32.
FID_HD double refine_start_distance(const MarkerRefineParams& rp) { return (double)(rp.min_rep_distance * rp.min_rep_distance + 1.f); }

// The largest squared distance between the predicted corners p and candidate c read from corner rot on (float32 differences and
// products, as Point2f).
FID_HD float refine_corner_distance(const float p[8], const float* c, int rot) {
    float best = 0.f;
    for (int k = 0; k < 4; k++) {
        const int q = (rot + k) & 3;
        const float dx = p[2 * k] - c[2 * q], dy = p[2 * k + 1] - c[2 * q + 1];
        const float d = dx * dx + dy * dy;
        best = d > best ? d : best;
    }
    return best;
}

// The rotation of candidate c kept against the running best `closest` (-1: none), and its distance.
FID_HD int refine_rotation(const float p[8], const float* c, int check_all_orders, double closest, double* dist) {
    int rot = -1;
    for (int r = 0; r < (check_all_orders ? 4 : 1); r++) {
        const double d = refine_corner_distance(p, c, r);
        if (d < closest) {
            rot = r;
            *dist = d;
        }
    }
    return rot;
}

// Whether any candidate not taken is within the start distance of p.  Taking candidates only removes them, so a marker without one
// can never be recovered.
FID_HD bool refine_has_candidate(const MarkerRefineParams& rp, const float p[8], int n_rej, const float* rej, const uint8_t* taken) {
    const double start = refine_start_distance(rp);
    double d;
    for (int j = 0; j < n_rej; j++)
        if (!taken[j] && refine_rotation(p, rej + 8 * j, rp.check_all_orders, start, &d) >= 0) return true;
    return false;
}

// Step "matching" for one undetected marker (id, predicted corners p): the index of the rejected candidate it takes (-1: none) and,
// in out, that candidate's corners in the kept rotation.  Lanes split the distance screen over the candidates; the candidates that
// pass it are then replayed in order, uniformly over the lanes, with the running best of the sequential rule.
template <class Lanes, class Img>
FID_HD int refine_match(const Lanes& L, const Img& gray, int W, int H, const DevParams& P, const unsigned long long* dict, const MarkerRefineParams& rp, int id,
                        const float p[8], int n_rej, const float* rej, const uint8_t* taken, uint8_t* img, int* hist, float out[8]) {
    double closest = refine_start_distance(rp);
    const int max_corr = (int)((double)P.max_correction_bits * (double)rp.error_correction_rate);
    int best = -1, best_rot = 0;
    for (int j0 = 0; j0 < n_rej; j0 += L.count()) {
        const int j = j0 + L.lane();
        double d;
        // the running best only decreases, so a candidate that fails the screen now fails it later in this pass too
        uint32_t near = L.ballot(j < n_rej && !taken[j] && refine_rotation(p, rej + 8 * j, rp.check_all_orders, closest, &d) >= 0);
        while (near) {
            const int jj = j0 + fid_ctz(near);
            near &= near - 1;
            const float* c = rej + 8 * jj;
            const int rot = refine_rotation(p, c, rp.check_all_orders, closest, &d);
            if (rot < 0) continue;
            if (rp.error_correction_rate >= 0.f) {
                if (id < 0 || id >= P.n_markers) continue;  // no code to compare with
                QuadF q;
                for (int k = 0; k < 4; k++) {
                    q.x[k] = c[2 * ((k + rot) & 3)];
                    q.y[k] = c[2 * ((k + rot) & 3) + 1];
                }
                const CellBits bits = extract_bits(L, gray, W, H, q, P, img, hist);
                L.sync();
                if (!bits.ok) continue;
                const unsigned long long x = dict[(size_t)id * 4] ^ inner_code(bits, P);
                if (fid_popc((uint32_t)x) + fid_popc((uint32_t)(x >> 32)) >= max_corr) continue;  // strictly below, unlike detection
            }
            best = jj;
            best_rot = rot;
            closest = d;
        }
    }
    if (best >= 0)
        for (int k = 0; k < 4; k++) {
            out[2 * k] = rej[8 * best + 2 * ((k + best_rot) & 3)];
            out[2 * k + 1] = rej[8 * best + 2 * ((k + best_rot) & 3) + 1];
        }
    return best;
}

// cornerSubPix of corner c of a recovered marker q, with the detector's window rule.  masks: windows 1..5 concatenated (the marker
// corners' table, zeroZone (-1, -1)); patch: (2 FID_SUBPIX_MAX_WIN + 3)^2 floats of scratch.
template <class Img>
FID_HD void refine_subpix_corner(const Img& gray, int W, int H, const DevParams& P, const float* masks, const float q[8], int c, float xy[2], float* patch) {
    QuadF qq;
    for (int k = 0; k < 4; k++) {
        qq.x[k] = q[2 * k];
        qq.y[k] = q[2 * k + 1];
    }
    const float module = quad_module_size(qq, P.marker_size, P.marker_border_bits);
    int win = round_half_even_to_int((double)((float)P.rel_refine_win * module));
    win = win < 1 ? 1 : win;
    win = win < P.refine_win ? win : P.refine_win;
    int off = 0;
    for (int w = 1; w < win; w++) off += (2 * w + 1) * (2 * w + 1);
    xy[0] = q[2 * c];
    xy[1] = q[2 * c + 1];
    corner_subpix(gray, W, H, &xy[0], &xy[1], win, masks + off, P.refine_max_iter, P.refine_min_acc * P.refine_min_acc, patch);
}

// Board marker `row` projected through the pose (R, p = rvec | tvec) with the camera, rounded to float32 (cv::projectPoints).
FID_HD void refine_project(const float* obj, int row, const double R[9], const double p[6], const Camera& cam, float out[8]) {
    for (int k = 0; k < 4; k++) {
        const float* o = obj + (size_t)row * 12 + 3 * k;
        double uv[2];
        project_point(o[0], o[1], o[2], R, nullptr, p, cam, uv, nullptr);
        out[2 * k] = (float)uv[0];
        out[2 * k + 1] = (float)uv[1];
    }
}

// Board marker `row` through the board homography (cv::perspectiveTransform of its float32 x, y).
FID_HD void refine_transform(const float* obj, int row, const double Hm[9], float out[8]) {
    for (int k = 0; k < 4; k++) charuco_apply(Hm, obj[(size_t)row * 12 + 3 * k], obj[(size_t)row * 12 + 3 * k + 1], out + 2 * k);
}

}  // namespace fid
