// One pose per marker board: cv::aruco::Board::matchImagePoints(corners, ids) followed by cv::solvePnP(obj, img, K, D, rvec, tvec,
// false, SOLVEPNP_ITERATIVE) of OpenCV 4.13 (cv::findExtrinsicCameraParams2, calib3d/src/calibration_base.cpp) over every matched
// point, then the reprojection error of getReprojectionError (aruco_detect.cpp:203-221) and the quaternion of :447-448.
//
//   0. matching: the detections in detection order; each whose id is on the board appends that board marker's 4 object points
//      (float32, as Board stores them) and its own 4 corners.  A repeated detection contributes twice, as in cv2.
//   1. undistort every matched corner (pnp.cuh, undistort_point).
//   2. planarity: centroid and 3x3 scatter of the matched object points, its SVD; W[2] / W[1] < 1e-3 = planar.  Chosen per
//      frame: one visible face of a 3-D board is planar.
//   3a. planar: rotate into the plane frame (Rt = the singular vectors, or I when the plane is already z = const; Tt = -Rt Mc),
//       cv::findHomography(method 0) from the plane coordinates onto the normalised points, both rounded to float32 as
//       findHomography converts them: normalised DLT (smallest eigenvector of the 9x9 L^T L) and, for more than 4 points, its
//       10-iteration LM refinement (cv::LMSolver); then pnp.cuh's column orthonormalisation, composed back with Rt / Tt.
//   3b. non-planar: needs >= 6 points (cv2 raises below; status -1).  DLT: smallest eigenvector of the 12x12 L^T L as [RR | t],
//       its sign by det(RR) < 0, R = the nearest rotation to RR, t scaled by |R| / |RR| (Frobenius).
//   4. Levenberg-Marquardt on the distorted reprojection error of all points, the CvLevMarq schedule of pnp.cuh (<= 20
//      iterations, FLT_EPSILON relative step).
//
// Every sum over points goes through board_sum: per-lane partial sums over the points lane, lane + 32, ..., then a fixed xor
// butterfly.  On the device the 32 lanes are a warp and everything else runs warp-uniformly (every lane computes the same
// value); the host build loops over 32 virtual lanes and butterflies in the same order.  Everything is double.
#pragma once
#include "pnp.cuh"

namespace fid {

#define FID_BOARD_LANES 32

struct BoardPoseOut {
    int status;  // 1 pose, 0 no board marker detected, -1 cv2.solvePnP raises (non-planar and fewer than 6 points, or a degenerate DLT)
    int n_markers, n_points;
    double rvec[3], tvec[3], quat[4];  // quat: x y z w
    double image_error;                // mean squared reprojection error, px^2
    int lm_iters;
};

// Sorted (id, marker index) table of a board: the position of id in keys[0..n), or -1.
FID_HD int board_find(const int32_t* keys, int n, int id) {
    int lo = 0, hi = n - 1;
    while (lo <= hi) {
        const int mid = (lo + hi) >> 1;
        const int k = keys[mid];
        if (k == id) return mid;
        if (k < id) lo = mid + 1;
        else hi = mid - 1;
    }
    return -1;
}

// Board::matchImagePoints, one detection after another (the host restatement the device's ballot prefix must equal).
// obj_out [4 n_markers][3], img_out [4 n_markers][2]; returns n_markers.
FID_HD int board_match(int n_det, const int32_t* det_ids, const float* det_corners, int n_board, const int32_t* keys, const int32_t* marker_of,
                       const float* board_obj, float* obj_out, float* img_out) {
    int m = 0;
    for (int j = 0; j < n_det; j++) {
        const int k = board_find(keys, n_board, det_ids[j]);
        if (k < 0) continue;
        const float* o = board_obj + (size_t)marker_of[k] * 12;
        for (int c = 0; c < 12; c++) obj_out[(size_t)m * 12 + c] = o[c];
        for (int c = 0; c < 8; c++) img_out[(size_t)m * 8 + c] = det_corners[(size_t)j * 8 + c];
        m++;
    }
    return m;
}

// out[k] = sum over the points i < n of term(i)[k], in the order described at the top of this file.  Device: called by all 32
// lanes of a warp together; every lane returns the same bits.
template <int K, class Term>
FID_HD void board_sum(int n, const Term& term, double out[K]) {
#if defined(__CUDA_ARCH__)
    double acc[K];
#pragma unroll
    for (int k = 0; k < K; k++) acc[k] = 0.0;
    for (int i = threadIdx.x & (FID_BOARD_LANES - 1); i < n; i += FID_BOARD_LANES) {
        double v[K];
        term(i, v);
#pragma unroll
        for (int k = 0; k < K; k++) acc[k] += v[k];
    }
#pragma unroll
    for (int off = FID_BOARD_LANES / 2; off > 0; off >>= 1)
#pragma unroll
        for (int k = 0; k < K; k++) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], off);
#pragma unroll
    for (int k = 0; k < K; k++) out[k] = acc[k];
#else
    double acc[FID_BOARD_LANES][K], nxt[FID_BOARD_LANES][K];
    for (int l = 0; l < FID_BOARD_LANES; l++) {
        for (int k = 0; k < K; k++) acc[l][k] = 0.0;
        for (int i = l; i < n; i += FID_BOARD_LANES) {
            double v[K];
            term(i, v);
            for (int k = 0; k < K; k++) acc[l][k] += v[k];
        }
    }
    for (int off = FID_BOARD_LANES / 2; off > 0; off >>= 1) {
        for (int l = 0; l < FID_BOARD_LANES; l++)
            for (int k = 0; k < K; k++) nxt[l][k] = acc[l][k] + acc[l ^ off][k];
        for (int l = 0; l < FID_BOARD_LANES; l++)
            for (int k = 0; k < K; k++) acc[l][k] = nxt[l][k];
    }
    for (int k = 0; k < K; k++) out[k] = acc[0][k];
#endif
}

// First point and stride of this lane for per-point work whose results only this lane reads again (board_sum's split).
FID_HD int board_lane0() {
#if defined(__CUDA_ARCH__)
    return threadIdx.x & (FID_BOARD_LANES - 1);
#else
    return 0;
#endif
}
FID_HD int board_lane_step() {
#if defined(__CUDA_ARCH__)
    return FID_BOARD_LANES;
#else
    return 1;
#endif
}

// cv::findHomography(src, dst, 0) for n >= 4 points given by pts(i, s[2], d[2]) as float32 (the conversion findHomography makes).
// Returns false where its kernel gives no model (a degenerate spread: no homography).
template <class Pts>
FID_HD bool board_homography(int n, const Pts& pts, double Hm[9]) {
    // HomographyEstimatorCallback::runKernel: centroids and mean absolute deviations, then the normalised DLT
    double c[4];
    board_sum<4>(n, [&](int i, double v[4]) {
        float s[2], d[2];
        pts(i, s, d);
        v[0] = d[0];
        v[1] = d[1];
        v[2] = s[0];
        v[3] = s[1];
    }, c);
    const double cmx = c[0] / n, cmy = c[1] / n, cMx = c[2] / n, cMy = c[3] / n;
    double sd[4];
    board_sum<4>(n, [&](int i, double v[4]) {
        float s[2], d[2];
        pts(i, s, d);
        v[0] = fabs(d[0] - cmx);
        v[1] = fabs(d[1] - cmy);
        v[2] = fabs(s[0] - cMx);
        v[3] = fabs(s[1] - cMy);
    }, sd);
    const double eps = 2.220446049250313e-16;
    if (fabs(sd[0]) < eps || fabs(sd[1]) < eps || fabs(sd[2]) < eps || fabs(sd[3]) < eps) return false;
    const double smx = n / sd[0], smy = n / sd[1], sMx = n / sd[2], sMy = n / sd[3];
    double ltl[45];  // upper triangle of L^T L, row by row
    board_sum<45>(n, [&](int i, double v[45]) {
        float s[2], d[2];
        pts(i, s, d);
        const double x = (d[0] - cmx) * smx, y = (d[1] - cmy) * smy;
        const double X = (s[0] - cMx) * sMx, Y = (s[1] - cMy) * sMy;
        const double Lx[9] = {X, Y, 1, 0, 0, 0, -x * X, -x * Y, -x};
        const double Ly[9] = {0, 0, 0, X, Y, 1, -y * X, -y * Y, -y};
        int o = 0;
        for (int j = 0; j < 9; j++)
            for (int k = j; k < 9; k++) v[o++] = Lx[j] * Lx[k] + Ly[j] * Ly[k];
    }, ltl);
    double LtL[9][9], w[9], V[9][9];
    for (int j = 0, o = 0; j < 9; j++)
        for (int k = j; k < 9; k++, o++) LtL[j][k] = LtL[k][j] = ltl[o];
    jacobi_eigen<9>(LtL, w, V);
    int best = 0;
    for (int i = 1; i < 9; i++)
        if (w[i] < w[best]) best = i;
    double H0[9];
    for (int i = 0; i < 9; i++) H0[i] = V[i][best];
    const double invHnorm[9] = {1.0 / smx, 0, cmx, 0, 1.0 / smy, cmy, 0, 0, 1};
    const double Hnorm2[9] = {sMx, 0, -cMx * sMx, 0, sMy, -cMy * sMy, 0, 0, 1};
    double T[9];
    mat3_mul(invHnorm, H0, T);
    mat3_mul(T, Hnorm2, Hm);
    const double inv = 1.0 / Hm[8];
    for (int i = 0; i < 9; i++) Hm[i] *= inv;
    if (n <= 4) return true;
    // HomographyRefineCallback under cv::LMSolver (10 iterations, eps FLT_EPSILON): lambda = 10^lg, lg from -3, -1 after an
    // accepted step (>= -16), +1 after a rejected one (<= 16; a rejection at 16 counts as an iteration)
    auto residual = [&](int i, const double h[8], double r[5]) {  // r = Mx ww, My ww, ww, xi, yi; returns the squared residual
        float s[2], d[2];
        pts(i, s, d);
        const double Mx = s[0], My = s[1];
        double ww = h[6] * Mx + h[7] * My + 1.;
        ww = fabs(ww) > eps ? 1. / ww : 0;
        const double xi = (h[0] * Mx + h[1] * My + h[2]) * ww;
        const double yi = (h[3] * Mx + h[4] * My + h[5]) * ww;
        r[0] = Mx * ww;
        r[1] = My * ww;
        r[2] = ww;
        r[3] = xi;
        r[4] = yi;
        return (xi - d[0]) * (xi - d[0]) + (yi - d[1]) * (yi - d[1]);
    };
    auto eval = [&](const double h[8], double v[45]) {  // J^T J upper triangle (36), J^T r (8), |r|^2
        board_sum<45>(n, [&](int i, double q[45]) {
            float s[2], d[2];
            pts(i, s, d);
            double r[5];
            q[44] = residual(i, h, r);
            const double ex = r[3] - d[0], ey = r[4] - d[1];
            const double Jx[8] = {r[0], r[1], r[2], 0, 0, 0, -r[0] * r[3], -r[1] * r[3]};
            const double Jy[8] = {0, 0, 0, r[0], r[1], r[2], -r[0] * r[4], -r[1] * r[4]};
            int o = 0;
            for (int a = 0; a < 8; a++)
                for (int b = a; b < 8; b++) q[o++] = Jx[a] * Jx[b] + Jy[a] * Jy[b];
            for (int a = 0; a < 8; a++) q[36 + a] = Jx[a] * ex + Jy[a] * ey;
        }, v);
    };
    double x[8], v[45];
    for (int k = 0; k < 8; k++) x[k] = Hm[k];
    eval(x, v);
    double S = v[44];
    int lg = -3, iter = 0;
    const double epsx = 1.1920928955078125e-07;
    for (;;) {
        double A[8][8], g[8], d[8], xd[8];
        const double lambda = exp(lg * 2.302585092994046);
        for (int a = 0, o = 0; a < 8; a++)
            for (int b = a; b < 8; b++, o++) A[a][b] = A[b][a] = v[o];
        for (int a = 0; a < 8; a++) {
            A[a][a] *= 1 + lambda;
            g[a] = v[36 + a];
        }
        solve_sym<8>(A, g, d);
        for (int a = 0; a < 8; a++) xd[a] = x[a] - d[a];
        double Sd;
        board_sum<1>(n, [&](int i, double q[1]) {
            double r[5];
            q[0] = residual(i, xd, r);
        }, &Sd);
        if (Sd < S) {
            S = Sd;
            lg = lg - 1 > -16 ? lg - 1 : -16;
            iter++;
            for (int a = 0; a < 8; a++) x[a] = xd[a];
            eval(x, v);
        } else {
            iter += lg == 16;
            lg = lg + 1 < 16 ? lg + 1 : 16;
        }
        double dn = 0.0;
        for (int a = 0; a < 8; a++) dn = fabs(d[a]) > dn ? fabs(d[a]) : dn;
        if (!(iter < 10 && dn >= epsx && S >= epsx * epsx)) break;
    }
    for (int k = 0; k < 8; k++) Hm[k] = x[k];
    Hm[8] = 1.0;
    return true;
}

// The sum of squared reprojection errors of the n points obj / img at p = {rvec, tvec}; f32: with the projections rounded to float
// (getReprojectionError).
FID_HD double board_sq_error(int n, const float* obj, const float* img, const Camera& cam, const double p[6], bool f32) {
    double R[9], s[1];
    rodrigues_v2m(p, R, nullptr);
    board_sum<1>(n, [&](int i, double v[1]) {
        double uv[2];
        project_point(obj[3 * i], obj[3 * i + 1], obj[3 * i + 2], R, nullptr, p, cam, uv, nullptr);
        if (f32) {
            const double e = dist2f(img[2 * i], img[2 * i + 1], (float)uv[0], (float)uv[1]);
            v[0] = e * e;
        } else {
            const double ex = uv[0] - img[2 * i], ey = uv[1] - img[2 * i + 1];
            v[0] = ex * ex + ey * ey;
        }
    }, s);
    return s[0];
}

// Step 4 of solvePnP(ITERATIVE) (cv::findExtrinsicCameraParams2's refinement; also all that solvePnP runs with
// useExtrinsicGuess): Levenberg-Marquardt on the distorted reprojection error of the n points from p = {rvec, tvec} (updated in
// place), the CvLevMarq schedule of pnp.cuh (<= 20 iterations, FLT_EPSILON relative step).  Returns the iterations.
FID_HD int board_pose_lm(int n, const float* obj, const float* img, const Camera& cam, double p[6]) {
    auto normal_eq = [&](const double q[6], double JtJ[6][6], double JtE[6], double* err2) {
        double R[9], dRdr[27], s[28];
        rodrigues_v2m(q, R, dRdr);
        board_sum<28>(n, [&](int i, double v[28]) {
            double uv[2], J[2][6];
            project_point(obj[3 * i], obj[3 * i + 1], obj[3 * i + 2], R, dRdr, q, cam, uv, J);
            const double ex = uv[0] - img[2 * i], ey = uv[1] - img[2 * i + 1];
            int o = 0;
            for (int a = 0; a < 6; a++)
                for (int b = a; b < 6; b++) v[o++] = J[0][a] * J[0][b] + J[1][a] * J[1][b];
            for (int a = 0; a < 6; a++) v[21 + a] = J[0][a] * ex + J[1][a] * ey;
            v[27] = ex * ex + ey * ey;
        }, s);
        for (int a = 0, o = 0; a < 6; a++)
            for (int b = a; b < 6; b++, o++) JtJ[a][b] = JtJ[b][a] = s[o];
        for (int a = 0; a < 6; a++) JtE[a] = s[21 + a];
        *err2 = s[27];
    };
    double JtJ[6][6], JtE[6], e2;
    normal_eq(p, JtJ, JtE, &e2);
    int lam = -3, iters = 0;
    double prev_err = sqrt(e2), en = 0.0;
    for (;;) {
        double prev[6];
        for (int a = 0; a < 6; a++) prev[a] = p[a];
        for (;;) {
            double A[6][6], delta[6];
            const double scale = 1.0 + exp(lam * 2.302585092994046);
            for (int a = 0; a < 6; a++)
                for (int b = 0; b < 6; b++) A[a][b] = a == b ? JtJ[a][b] * scale : JtJ[a][b];
            solve_sym6(A, JtE, delta);
            for (int a = 0; a < 6; a++) p[a] = prev[a] - delta[a];
            en = sqrt(board_sq_error(n, obj, img, cam, p, false));
            if (en > prev_err) {
                lam++;
                if (lam <= 16) continue;
            }
            break;
        }
        lam = lam - 1 > -16 ? lam - 1 : -16;
        iters++;
        double dn = 0.0, pn = 0.0;
        for (int a = 0; a < 6; a++) {
            dn += (p[a] - prev[a]) * (p[a] - prev[a]);
            pn += prev[a] * prev[a];
        }
        if (iters >= 20 || sqrt(dn) / sqrt(pn) < 1.1920928955078125e-07) break;
        prev_err = en;
        normal_eq(p, JtJ, JtE, &e2);
    }
    return iters;
}

// solvePnP(ITERATIVE) of n matched points: obj [n][3] float32 (metres), img [n][2] float32 (px); mn [n][2] is scratch for the
// normalised points (each lane writes and reads only its own points).  Fills everything of out but n_markers.
FID_HD void solve_board_pose(int n, const float* obj, const float* img, double* mn, const Camera& cam, BoardPoseOut* out) {
    out->status = 0;
    out->n_points = n;
    out->image_error = 0.0;
    out->lm_iters = 0;
    for (int k = 0; k < 3; k++) out->rvec[k] = out->tvec[k] = 0.0;
    for (int k = 0; k < 4; k++) out->quat[k] = 0.0;
    if (n <= 0) return;
    // 1. normalise + undistort
    for (int i = board_lane0(); i < n; i += board_lane_step()) undistort_point(img[2 * i], img[2 * i + 1], cam, mn + 2 * i);
    // 2. planarity of the matched object points
    double msum[3];
    board_sum<3>(n, [&](int i, double v[3]) {
        for (int k = 0; k < 3; k++) v[k] = obj[3 * i + k];
    }, msum);
    const double Mc[3] = {msum[0] * (1.0 / n), msum[1] * (1.0 / n), msum[2] * (1.0 / n)};
    double mm[6];
    board_sum<6>(n, [&](int i, double v[6]) {
        const double a = obj[3 * i] - Mc[0], b = obj[3 * i + 1] - Mc[1], c = obj[3 * i + 2] - Mc[2];
        v[0] = a * a;
        v[1] = a * b;
        v[2] = a * c;
        v[3] = b * b;
        v[4] = b * c;
        v[5] = c * c;
    }, mm);
    double MM[3][3] = {{mm[0], mm[1], mm[2]}, {mm[1], mm[3], mm[4]}, {mm[2], mm[4], mm[5]}}, ew[3], EV[3][3];
    jacobi_eigen<3>(MM, ew, EV);
    int ord[3] = {0, 1, 2};  // singular values (|eigenvalues|) in descending order
    for (int a = 0; a < 3; a++)
        for (int b = a + 1; b < 3; b++)
            if (fabs(ew[ord[b]]) > fabs(ew[ord[a]])) {
                const int t = ord[a];
                ord[a] = ord[b];
                ord[b] = t;
            }
    double p[6];
    if (fabs(ew[ord[2]]) / fabs(ew[ord[1]]) < 1e-3) {
        // 3a. planar.  Rt: rows = the singular vectors (cvSVD's V^T), I when the plane is already z = const, det +1
        double Rt[9];
        for (int r = 0; r < 3; r++)
            for (int k = 0; k < 3; k++) Rt[3 * r + k] = EV[k][ord[r]];
        if (Rt[2] * Rt[2] + Rt[5] * Rt[5] < 1e-10)
            for (int k = 0; k < 9; k++) Rt[k] = (k % 4 == 0) ? 1.0 : 0.0;
        const double det = Rt[0] * (Rt[4] * Rt[8] - Rt[5] * Rt[7]) - Rt[1] * (Rt[3] * Rt[8] - Rt[5] * Rt[6]) + Rt[2] * (Rt[3] * Rt[7] - Rt[4] * Rt[6]);
        if (det < 0)
            for (int k = 0; k < 9; k++) Rt[k] = -Rt[k];
        double Tt[3];
        for (int r = 0; r < 3; r++) Tt[r] = -(Rt[3 * r] * Mc[0] + Rt[3 * r + 1] * Mc[1] + Rt[3 * r + 2] * Mc[2]);
        double Hm[9];
        const bool ok = board_homography(n, [&](int i, float s[2], float d[2]) {
            const double X = obj[3 * i], Y = obj[3 * i + 1], Z = obj[3 * i + 2];
            s[0] = (float)(Rt[0] * X + Rt[1] * Y + Rt[2] * Z + Tt[0]);
            s[1] = (float)(Rt[3] * X + Rt[4] * Y + Rt[5] * Z + Tt[1]);
            d[0] = (float)mn[2 * i];
            d[1] = (float)mn[2 * i + 1];
        }, Hm);
        bool finite = ok;
        for (int k = 0; k < 9; k++) finite = finite && isfinite(Hm[k]);
        double Rm[9];
        if (finite) {
            double h1[3] = {Hm[0], Hm[3], Hm[6]}, h2[3] = {Hm[1], Hm[4], Hm[7]};
            const double h3[3] = {Hm[2], Hm[5], Hm[8]};
            const double n1 = sqrt(h1[0] * h1[0] + h1[1] * h1[1] + h1[2] * h1[2]);
            const double n2 = sqrt(h2[0] * h2[0] + h2[1] * h2[1] + h2[2] * h2[2]);
            const double eps = 2.220446049250313e-16;
            const double d1 = 1.0 / (n1 > eps ? n1 : eps), d2 = 1.0 / (n2 > eps ? n2 : eps);
            const double d3 = 2.0 / ((n1 + n2) > eps ? (n1 + n2) : eps);
            for (int k = 0; k < 3; k++) {
                h1[k] *= d1;
                h2[k] *= d2;
            }
            double t0[3] = {h3[0] * d3, h3[1] * d3, h3[2] * d3};
            const double hx[3] = {h1[1] * h2[2] - h1[2] * h2[1], h1[2] * h2[0] - h1[0] * h2[2], h1[0] * h2[1] - h1[1] * h2[0]};
            const double Rh[9] = {h1[0], h2[0], hx[0], h1[1], h2[1], hx[1], h1[2], h2[2], hx[2]};
            double r0[3], Rr[9];
            rodrigues_m2v(Rh, r0);
            rodrigues_v2m(r0, Rr, nullptr);
            for (int k = 0; k < 3; k++) p[3 + k] = Rr[3 * k] * Tt[0] + Rr[3 * k + 1] * Tt[1] + Rr[3 * k + 2] * Tt[2] + t0[k];
            mat3_mul(Rr, Rt, Rm);
        } else {  // no homography: the identity and zero translation, as findExtrinsicCameraParams2
            for (int k = 0; k < 9; k++) Rm[k] = (k % 4 == 0) ? 1.0 : 0.0;
            p[3] = p[4] = p[5] = 0.0;
        }
        rodrigues_m2v(Rm, p);
    } else {
        // 3b. non-planar: DLT
        if (n < 6) {
            out->status = -1;
            return;
        }
        double ll[78];  // upper triangle of the 12x12 L^T L
        board_sum<78>(n, [&](int i, double v[78]) {
            const double X = obj[3 * i], Y = obj[3 * i + 1], Z = obj[3 * i + 2], x = -mn[2 * i], y = -mn[2 * i + 1];
            const double La[12] = {X, Y, Z, 1., 0., 0., 0., 0., x * X, x * Y, x * Z, x};
            const double Lb[12] = {0., 0., 0., 0., X, Y, Z, 1., y * X, y * Y, y * Z, y};
            int o = 0;
            for (int j = 0; j < 12; j++)
                for (int k = j; k < 12; k++) v[o++] = La[j] * La[k] + Lb[j] * Lb[k];
        }, ll);
        double LL[12][12], lw[12], LV[12][12];
        for (int j = 0, o = 0; j < 12; j++)
            for (int k = j; k < 12; k++, o++) LL[j][k] = LL[k][j] = ll[o];
        jacobi_eigen<12>(LL, lw, LV);
        int best = 0;
        for (int i = 1; i < 12; i++)
            if (fabs(lw[i]) < fabs(lw[best])) best = i;
        double RR[9], tt[3];
        for (int r = 0; r < 3; r++) {
            for (int k = 0; k < 3; k++) RR[3 * r + k] = LV[4 * r + k][best];
            tt[r] = LV[4 * r + 3][best];
        }
        const double det = RR[0] * (RR[4] * RR[8] - RR[5] * RR[7]) - RR[1] * (RR[3] * RR[8] - RR[5] * RR[6]) + RR[2] * (RR[3] * RR[7] - RR[4] * RR[6]);
        if (det < 0) {
            for (int k = 0; k < 9; k++) RR[k] = -RR[k];
            for (int k = 0; k < 3; k++) tt[k] = -tt[k];
        }
        double sc = 0.0;
        for (int k = 0; k < 9; k++) sc += RR[k] * RR[k];
        sc = sqrt(sc);
        if (!(fabs(sc) > 2.220446049250313e-16)) {  // CV_Assert in findExtrinsicCameraParams2
            out->status = -1;
            return;
        }
        double Rm[9];
        for (int k = 0; k < 9; k++) Rm[k] = RR[k];
        orthonormalize3(Rm);
        double rn = 0.0;
        for (int k = 0; k < 9; k++) rn += Rm[k] * Rm[k];
        const double f = sqrt(rn) / sc;
        for (int k = 0; k < 3; k++) p[3 + k] = tt[k] * f;
        rodrigues_m2v(Rm, p);
    }
    // 4. Levenberg-Marquardt (CvLevMarq schedule, as solve_marker_pose)
    const int iters = board_pose_lm(n, obj, img, cam, p);
    out->status = 1;
    out->lm_iters = iters;
    for (int k = 0; k < 3; k++) {
        out->rvec[k] = p[k];
        out->tvec[k] = p[3 + k];
    }
    // reprojection error with the projections rounded to float32 (getReprojectionError :208-219, over all matched points)
    out->image_error = board_sq_error(n, obj, img, cam, p, true) / n;
    // quaternion (:447-448)
    const double angle = sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]);
    const double ax = p[0] / angle, ay = p[1] / angle, az = p[2] / angle;
    const double dlen = sqrt(ax * ax + ay * ay + az * az);
    const double s = sin(angle * 0.5) / dlen;
    out->quat[0] = ax * s;
    out->quat[1] = ay * s;
    out->quat[2] = az * s;
    out->quat[3] = cos(angle * 0.5);
}

}  // namespace fid
