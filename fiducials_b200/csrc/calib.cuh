// Camera calibration from views of a planar (or, with an intrinsic guess, any) rig: cv::calibrateCameraExtended of OpenCV 4.13
// (calib3d/src/calibration.cpp, cvCalibrateCamera2Internal) for the camera model of fid_camera, K = [fx 0 cx; 0 fy cy; 0 0 1]
// and the plumb_bob coefficients k1 k2 p1 p2 k3.
//
//   1. input: per view n >= 4 object points and image points, float32 as cv2 takes them; converted to double (exact).  Without
//      CALIB_USE_INTRINSIC_GUESS the rig must be planar (mean and standard deviation of every z within 1e-5) and every z is set
//      to 0.  The checks and the conversion are the host's (fid_calibrate_camera).
//   2. initial intrinsics, without a guess (cvInitIntrinsicParams2D): per view cv::findHomography(method 0) from the object
//      plane (X, Y) onto the image points (board_pnp.cuh, board_homography; a degenerate spread raises in cv2), minus the
//      principal point ((w - 1) / 2, (h - 1) / 2); the two vanishing-point rows of the view (calib_view_homography); then
//      the 2x2 normal equations summed over the views in view order, solved, f = sqrt(|1 / x|) (calib_init_intrinsics);
//      FIX_ASPECT_RATIO replaces fx, fy by aspect * t, t with t = (fx + fy) / (aspect + 1).
//   3. initial extrinsics: cv::findExtrinsicCameraParams2 per view with the initial K and D (board_pnp.cuh, solve_board_pose).
//   4. joint Levenberg-Marquardt, the CvLevMarq::updateAlt schedule: lambda = 10^lg, lg from -3; every J evaluation at the
//      current parameters p is followed by trial steps p' = p - (J^T J + lambda diag(J^T J))^-1 J^T e over the free parameters;
//      a trial whose error exceeds the previous one raises lg and is retried from the same J while lg <= 16 (a trial at lg 17
//      is kept anyway); every kept trial lowers lg (>= -16) and counts one iteration; stop after max_iter iterations or when
//      |p' - p| / (|p| + DBL_EPSILON) < epsilon.  The normal equations are not formed densely: per view the blocks
//      U_i = Ji^T Ji (9x9), W_i = Ji^T Je (9x6), V_i = Je^T Je (6x6), gi_i, ge_i and the cost (calib_view_eval); the damped
//      step is the Schur complement S = sum U (damped) - sum W_i Vd_i^-1 W_i^T over the free intrinsics (calib_view_schur,
//      calib_solve_intrinsics) and the back-substituted per-view step (calib_view_trial) -- the same step cv2 solves densely.
//      FIX_ASPECT_RATIO keeps fx = aspect * fy with fy free (d u / d fy = aspect xd).
//   5. outputs at the final parameters: rms = sqrt(sum e^2 / total), per view sqrt(sum_view e^2 / n_view), and the standard
//      deviations sqrt(diag((J^T J)^-1) sigma^2), sigma^2 = sum e^2 / (total - free parameters), from the undamped blocks:
//      S^-1 for the intrinsics and V_i^-1 + V_i^-1 W_i^T S^-1 W_i V_i^-1 per view (calib_view_std).
//
// Every sum over the points of a view goes through board_sum (a fixed order); every sum over views runs in view order.  The
// functions are shared by the sm_90a kernels (fid_calib.cu) and the host build, and cos, sin, acos and exp -- in the headers
// below too -- are the polynomial ones of this file, so that host and device compute the same bits.
#pragma once
#if defined(FID_HD)
#error "calib.cuh must be the first fiducials header of its translation unit (it gives pnp.cuh / board_pnp.cuh their cos, sin, acos and exp)"
#endif
#include "common.cuh"

namespace fid {

// ---- deterministic elementary functions (only +, -, *, /, sqrt, rint and ldexp, all exact or correctly rounded) ------------
FID_HD double det_exp(double x) {
    // x = k ln2 + r, |r| <= ln2 / 2 (ln2 in two parts, the first with 21 trailing zero bits); e^r by Horner to r^17 / 17!
    const double ln2_hi = 6.93147180369123816490e-01, ln2_lo = 1.90821492927058770002e-10;
    const double k = rint(x * 1.44269504088896338700e+00);
    const double r = (x - k * ln2_hi) - k * ln2_lo;
    double s = 1.0;
    for (int i = 17; i >= 1; i--) s = 1.0 + s * r / i;
    return ldexp(s, (int)k);
}
FID_HD void det_sincos(double x, double* sn, double* cs) {
    // x = q pi/2 + r, |r| <= pi/4 (pi/2 in two parts, the first with 33 significant bits); Taylor series of sin r and cos r
    const double q = rint(x * 6.36619772367581382433e-01);
    const double r = (x - q * 1.57079632673412561417e+00) - q * 6.07710050650619224932e-11, r2 = r * r;
    double s = 1.0, c = 1.0;
    for (int i = 22; i >= 2; i -= 2) {
        s = 1.0 - s * r2 / (double)(i * (i + 1));
        c = 1.0 - c * r2 / (double)((i - 1) * i);
    }
    s *= r;
    const long long quad = (long long)q & 3;
    *sn = quad == 0 ? s : (quad == 1 ? c : (quad == 2 ? -s : -c));
    *cs = quad == 0 ? c : (quad == 1 ? -s : (quad == 2 ? -c : s));
}
FID_HD double det_atan01(double t) {  // atan(t), 0 <= t <= 1
    const double pi4 = 7.85398163397448278999e-01;
    const bool big = t > 0.41421356237309503;  // atan t = pi/4 + atan((t - 1) / (t + 1))
    const double u = big ? (t - 1.0) / (t + 1.0) : t, u2 = u * u;
    double s = 1.0 / 47.0;
    for (int k = 22; k >= 0; k--) s = 1.0 / (2 * k + 1) - u2 * s;
    return big ? pi4 + u * s : u * s;
}
FID_HD double det_acos(double c) {  // acos c = 2 atan(sqrt(1 - c) / sqrt(1 + c))
    const double a = sqrt(1.0 - c), b = sqrt(1.0 + c);
    return a <= b ? 2.0 * det_atan01(a / b) : 3.14159265358979311600e+00 - 2.0 * det_atan01(b / a);
}
// The names pnp.cuh and board_pnp.cuh call: unqualified calls inside namespace fid find these before the global libm ones.
FID_HD double exp(double x) { return det_exp(x); }
FID_HD double sin(double x) {
    double s, c;
    det_sincos(x, &s, &c);
    return s;
}
FID_HD double cos(double x) {
    double s, c;
    det_sincos(x, &s, &c);
    return c;
}
FID_HD double acos(double x) { return det_acos(x); }

}  // namespace fid

#include "board_pnp.cuh"

namespace fid {

// cv2's CALIB_* values
#define FID_CALIB_USE_INTRINSIC_GUESS_ 0x00001
#define FID_CALIB_FIX_ASPECT_RATIO_ 0x00002
#define FID_CALIB_FIX_PRINCIPAL_POINT_ 0x00004
#define FID_CALIB_ZERO_TANGENT_DIST_ 0x00008
#define FID_CALIB_FIX_FOCAL_LENGTH_ 0x00010
#define FID_CALIB_FIX_K1_ 0x00020
#define FID_CALIB_FIX_K2_ 0x00040
#define FID_CALIB_FIX_K3_ 0x00080

// Per-view block layout (doubles): U upper 45, W 9x6 row-major 54, V upper 21, gi 9, ge 6, cost 1
#define CALIB_U 0
#define CALIB_W 45
#define CALIB_V 99
#define CALIB_GI 120
#define CALIB_GE 129
#define CALIB_COST 135
#define CALIB_BLK 136
// Per-view Schur layout: Vd^-1 6x6 36, Q = W Vd^-1 W^T upper 45, q = W Vd^-1 ge 9
#define CALIB_VINV 0
#define CALIB_Q 36
#define CALIB_QV 81
#define CALIB_SCH 90
#define CALIB_MAX_STEPS 2048  // trial steps of one run: <= 2 max_iter + 20 (max_iter <= 1000)

// The free-parameter mask of the intrinsics fx fy cx cy k1 k2 p1 p2 k3 (CvLevMarq's mask[0..8]).
FID_HD void calib_mask(int flags, int mask[9]) {
    for (int a = 0; a < 9; a++) mask[a] = 1;
    if (flags & FID_CALIB_FIX_ASPECT_RATIO_) mask[0] = 0;
    if (flags & FID_CALIB_FIX_FOCAL_LENGTH_) mask[0] = mask[1] = 0;
    if (flags & FID_CALIB_FIX_PRINCIPAL_POINT_) mask[2] = mask[3] = 0;
    if (flags & FID_CALIB_ZERO_TANGENT_DIST_) mask[6] = mask[7] = 0;
    if (flags & FID_CALIB_FIX_K1_) mask[4] = 0;
    if (flags & FID_CALIB_FIX_K2_) mask[5] = 0;
    if (flags & FID_CALIB_FIX_K3_) mask[8] = 0;
}

FID_HD Camera calib_camera(const double in[9]) { return Camera{in[0], in[1], in[2], in[3], in[4], in[5], in[6], in[7], in[8]}; }

// Stage 2, one view: its homography and the two rows (Ap[4], bp[2]) of the vanishing-point system; false if cv2 raises.
FID_HD bool calib_view_homography(int n, const float* obj, const float* img, double cx, double cy, double ab[6]) {
    double H[9];
    const bool ok = board_homography(n, [&](int i, float s[2], float d[2]) {
        s[0] = obj[3 * i];
        s[1] = obj[3 * i + 1];
        d[0] = img[2 * i];
        d[1] = img[2 * i + 1];
    }, H);
    if (!ok) return false;
    H[0] -= H[6] * cx;
    H[1] -= H[7] * cx;
    H[2] -= H[8] * cx;
    H[3] -= H[6] * cy;
    H[4] -= H[7] * cy;
    H[5] -= H[8] * cy;
    double h[3], v[3], d1[3], d2[3], nn[4] = {0, 0, 0, 0};
    for (int j = 0; j < 3; j++) {
        const double t0 = H[j * 3], t1 = H[j * 3 + 1];
        h[j] = t0;
        v[j] = t1;
        d1[j] = (t0 + t1) * 0.5;
        d2[j] = (t0 - t1) * 0.5;
        nn[0] += t0 * t0;
        nn[1] += t1 * t1;
        nn[2] += d1[j] * d1[j];
        nn[3] += d2[j] * d2[j];
    }
    for (int j = 0; j < 4; j++) nn[j] = 1. / sqrt(nn[j]);
    for (int j = 0; j < 3; j++) {
        h[j] *= nn[0];
        v[j] *= nn[1];
        d1[j] *= nn[2];
        d2[j] *= nn[3];
    }
    ab[0] = h[0] * v[0];
    ab[1] = h[1] * v[1];
    ab[2] = d1[0] * d2[0];
    ab[3] = d1[1] * d2[1];
    ab[4] = -h[2] * v[2];
    ab[5] = -d1[2] * d2[2];
    return true;
}

// The 2x2 normal-equation terms of one view's rows (summed over views in view order).
FID_HD void calib_view_normal2(const double ab[6], double t[5]) {
    t[0] = ab[0] * ab[0] + ab[2] * ab[2];
    t[1] = ab[0] * ab[1] + ab[2] * ab[3];
    t[2] = ab[1] * ab[1] + ab[3] * ab[3];
    t[3] = ab[0] * ab[4] + ab[2] * ab[5];
    t[4] = ab[1] * ab[4] + ab[3] * ab[5];
}

// Stage 2, all views: intrinsics fx fy cx cy from the summed terms; aspect 0 = free aspect ratio.
FID_HD void calib_init_intrinsics(const double t[5], int width, int height, double aspect, double A[4]) {
    const double M[2][2] = {{t[0], t[1]}, {t[1], t[2]}}, b[2] = {t[3], t[4]};
    double f[2];
    solve_sym<2>(M, b, f);
    A[0] = sqrt(fabs(1. / f[0]));
    A[1] = sqrt(fabs(1. / f[1]));
    if (aspect != 0) {
        const double tf = (A[0] + A[1]) / (aspect + 1.);
        A[0] = aspect * tf;
        A[1] = tf;
    }
    A[2] = (width - 1) * 0.5;
    A[3] = (height - 1) * 0.5;
}

// One point: residual e = projection - image point, and its Jacobian over the 9 intrinsics and the view's 6 extrinsics
// (cvProjectPoints2Internal's dpdf / dpdc / dpdk / dpdr / dpdt).
template <class T>
FID_HD void calib_point(const T* o, const float* m, const double in[9], double aspect, const double R[9], const double* dRdr, const double p[6],
                        double e[2], double Ji[2][9], double Je[2][6]) {
    const Camera cam = calib_camera(in);
    double uv[2];
    project_point(o[0], o[1], o[2], R, dRdr, p, cam, uv, Je);
    e[0] = uv[0] - m[0];
    e[1] = uv[1] - m[1];
    if (!Ji) return;
    double x = R[0] * o[0] + R[1] * o[1] + R[2] * o[2] + p[3];
    double y = R[3] * o[0] + R[4] * o[1] + R[5] * o[2] + p[4];
    double z = R[6] * o[0] + R[7] * o[1] + R[8] * o[2] + p[5];
    z = z != 0.0 ? 1.0 / z : 1.0;
    x *= z;
    y *= z;
    const double r2 = x * x + y * y, r4 = r2 * r2, r6 = r4 * r2;
    const double a1 = 2 * x * y, a2 = r2 + 2 * x * x, a3 = r2 + 2 * y * y;
    const double cdist = 1 + cam.k1 * r2 + cam.k2 * r4 + cam.k3 * r6;
    const double xd = x * cdist + cam.p1 * a1 + cam.p2 * a2, yd = y * cdist + cam.p1 * a3 + cam.p2 * a1;
    const double ju[9] = {aspect != 0 ? 0.0 : xd, aspect != 0 ? xd * aspect : 0.0, 1, 0, cam.fx * x * r2, cam.fx * x * r4, cam.fx * a1, cam.fx * a2,
                          cam.fx * x * r6};
    const double jv[9] = {0, yd, 0, 1, cam.fy * y * r2, cam.fy * y * r4, cam.fy * a3, cam.fy * a1, cam.fy * y * r6};
    for (int a = 0; a < 9; a++) {
        Ji[0][a] = ju[a];
        Ji[1][a] = jv[a];
    }
}

// Stage 4, one view: the blocks U, W, V, gi, ge and the cost at intrinsics `in` and extrinsics p (layout CALIB_*).
template <class T>
FID_HD void calib_view_eval(int n, const T* obj, const float* img, const double in[9], double aspect, const double p[6], double* blk) {
    double R[9], dRdr[27];
    rodrigues_v2m(p, R, dRdr);
    auto point = [&](int i, double e[2], double Ji[2][9], double Je[2][6]) { calib_point(obj + 3 * i, img + 2 * i, in, aspect, R, dRdr, p, e, Ji, Je); };
    double s1[37];  // V 21, gi 9, ge 6, cost 1
    board_sum<37>(n, [&](int i, double v[37]) {
        double e[2], Ji[2][9], Je[2][6];
        point(i, e, Ji, Je);
        int o = 0;
        for (int a = 0; a < 6; a++)
            for (int b = a; b < 6; b++) v[o++] = Je[0][a] * Je[0][b] + Je[1][a] * Je[1][b];
        for (int a = 0; a < 9; a++) v[o++] = Ji[0][a] * e[0] + Ji[1][a] * e[1];
        for (int a = 0; a < 6; a++) v[o++] = Je[0][a] * e[0] + Je[1][a] * e[1];
        v[o] = e[0] * e[0] + e[1] * e[1];
    }, s1);
    for (int k = 0; k < 21; k++) blk[CALIB_V + k] = s1[k];
    for (int k = 0; k < 9; k++) blk[CALIB_GI + k] = s1[21 + k];
    for (int k = 0; k < 6; k++) blk[CALIB_GE + k] = s1[30 + k];
    blk[CALIB_COST] = s1[36];
    double s2[45];
    board_sum<45>(n, [&](int i, double v[45]) {
        double e[2], Ji[2][9], Je[2][6];
        point(i, e, Ji, Je);
        int o = 0;
        for (int a = 0; a < 9; a++)
            for (int b = a; b < 9; b++) v[o++] = Ji[0][a] * Ji[0][b] + Ji[1][a] * Ji[1][b];
    }, s2);
    for (int k = 0; k < 45; k++) blk[CALIB_U + k] = s2[k];
    double s3[54];
    board_sum<54>(n, [&](int i, double v[54]) {
        double e[2], Ji[2][9], Je[2][6];
        point(i, e, Ji, Je);
        for (int a = 0; a < 9; a++)
            for (int b = 0; b < 6; b++) v[6 * a + b] = Ji[0][a] * Je[0][b] + Ji[1][a] * Je[1][b];
    }, s3);
    for (int k = 0; k < 54; k++) blk[CALIB_W + k] = s3[k];
}

// Stage 4, one view: Vd^-1 (V with its diagonal times `scale` = 1 + lambda), Q = W Vd^-1 W^T and q = W Vd^-1 ge.
FID_HD void calib_view_schur(const double* blk, double scale, double* sch) {
    double Vd[6][6];
    for (int a = 0, o = 0; a < 6; a++)
        for (int b = a; b < 6; b++, o++) Vd[a][b] = Vd[b][a] = blk[CALIB_V + o];
    for (int a = 0; a < 6; a++) Vd[a][a] *= scale;
    double Vi[6][6];
    for (int c = 0; c < 6; c++) {
        double u[6] = {0, 0, 0, 0, 0, 0}, x[6];
        u[c] = 1.0;
        solve_sym<6>(Vd, u, x);
        for (int r = 0; r < 6; r++) Vi[r][c] = x[r];
    }
    for (int r = 0; r < 6; r++)
        for (int c = 0; c < 6; c++) sch[CALIB_VINV + 6 * r + c] = Vi[r][c];
    double Y[9][6];
    for (int a = 0; a < 9; a++)
        for (int j = 0; j < 6; j++) {
            double s = 0.0;
            for (int k = 0; k < 6; k++) s += blk[CALIB_W + 6 * a + k] * Vi[k][j];
            Y[a][j] = s;
        }
    for (int a = 0, o = 0; a < 9; a++)
        for (int b = a; b < 9; b++, o++) {
            double s = 0.0;
            for (int j = 0; j < 6; j++) s += Y[a][j] * blk[CALIB_W + 6 * b + j];
            sch[CALIB_Q + o] = s;
        }
    for (int a = 0; a < 9; a++) {
        double s = 0.0;
        for (int j = 0; j < 6; j++) s += Y[a][j] * blk[CALIB_GE + j];
        sch[CALIB_QV + a] = s;
    }
}

// The reduced intrinsic system S = U (diagonal times scale) - Q, r = g - q over the free parameters; a fixed parameter's row
// and column are replaced by the largest diagonal entry so that its solution is exactly 0.
FID_HD void calib_schur_system(const double U[45], const double g[9], const double Q[45], const double q[9], double scale, const int mask[9], double S[9][9],
                               double r[9]) {
    for (int a = 0, o = 0; a < 9; a++)
        for (int b = a; b < 9; b++, o++) S[a][b] = S[b][a] = (a == b ? U[o] * scale : U[o]) - Q[o];
    double dmax = 0.0;
    for (int a = 0; a < 9; a++)
        if (mask[a] && fabs(S[a][a]) > dmax) dmax = fabs(S[a][a]);
    if (dmax == 0.0) dmax = 1.0;
    for (int a = 0; a < 9; a++) {
        r[a] = mask[a] ? g[a] - q[a] : 0.0;
        if (mask[a]) continue;
        for (int b = 0; b < 9; b++) S[a][b] = S[b][a] = 0.0;
        S[a][a] = dmax;
    }
}

// Stage 4: the intrinsic step d (0 for fixed parameters).
FID_HD void calib_solve_intrinsics(const double U[45], const double g[9], const double Q[45], const double q[9], double scale, const int mask[9], double d[9]) {
    double S[9][9], r[9];
    calib_schur_system(U, g, Q, q, scale, mask, S, r);
    solve_sym<9>(S, r, d);
    for (int a = 0; a < 9; a++)
        if (!mask[a]) d[a] = 0.0;
}

// One view's cost sum e^2 at intrinsics `in`, extrinsics p and object points obj.
template <class T>
FID_HD double calib_view_cost(int n, const T* obj, const float* img, const double in[9], double aspect, const double p[6]) {
    double R[9];
    rodrigues_v2m(p, R, nullptr);
    double c;
    board_sum<1>(n, [&](int i, double v[1]) {
        double e[2];
        calib_point(obj + 3 * i, img + 2 * i, in, aspect, R, nullptr, p, e, nullptr, nullptr);
        v[0] = e[0] * e[0] + e[1] * e[1];
    }, &c);
    return c;
}

// Stage 4, one view: the back-substituted extrinsic step, the trial parameters p = pp - d and, at the trial intrinsics `in`,
// out = {cost, |p - pp|^2, |pp|^2}.
FID_HD void calib_view_trial(int n, const float* obj, const float* img, const double in[9], double aspect, const double* blk, const double* sch,
                             const double dint[9], const double pp[6], double p[6], double out[3]) {
    double r[6];
    for (int k = 0; k < 6; k++) {
        double s = blk[CALIB_GE + k];
        for (int a = 0; a < 9; a++) s -= blk[CALIB_W + 6 * a + k] * dint[a];
        r[k] = s;
    }
    double dn = 0.0, pn = 0.0;
    for (int j = 0; j < 6; j++) {
        double s = 0.0;
        for (int k = 0; k < 6; k++) s += sch[CALIB_VINV + 6 * j + k] * r[k];
        p[j] = pp[j] - s;
        dn += (p[j] - pp[j]) * (p[j] - pp[j]);
        pn += pp[j] * pp[j];
    }
    out[0] = calib_view_cost(n, obj, img, in, aspect, p);
    out[1] = dn;
    out[2] = pn;
}

// CvLevMarq (updateAlt) state of one run.
struct CalibLM {
    int state;  // 0 evaluate J at p, 1 trial step from the last J, 2 done
    int lg, iters, max_iter, n_steps, n_evals;
    double eps, err, prev_err;
    double aspect;
    int mask[9];
    double in[9], in_prev[9], dint[9];
    double U[45], g[9];  // sums over the views of the last J
    unsigned char steps[CALIB_MAX_STEPS];  // per trial: 1 kept, 0 rejected
};

FID_HD double calib_pow10(int lg) {  // 10^lg by exact-order multiplication (host and device agree)
    double s = 1.0;
    for (int k = 0; k < (lg < 0 ? -lg : lg); k++) s *= 10.0;
    return lg < 0 ? 1.0 / s : s;
}

FID_HD void calib_lm_init(CalibLM* s, const double in[9], int flags, double aspect, int max_iter, double eps) {
    s->state = 0;
    s->lg = -3;
    s->iters = s->n_steps = s->n_evals = 0;
    s->max_iter = max_iter;
    s->eps = eps;
    s->err = s->prev_err = 0.0;
    s->aspect = aspect;
    calib_mask(flags, s->mask);
    for (int a = 0; a < 9; a++) s->in[a] = s->in_prev[a] = in[a];
    if (flags & FID_CALIB_ZERO_TANGENT_DIST_) s->in[6] = s->in[7] = 0.0;
    if (aspect != 0) s->in[0] = s->in[1] * aspect;
}

// After a J evaluation: the sums of the views' U, gi and costs (in view order) are in s->U, s->g and err.
FID_HD void calib_lm_after_eval(CalibLM* s, double err) {
    s->n_evals++;
    s->err = s->prev_err = err;
    for (int a = 0; a < 9; a++) s->in_prev[a] = s->in[a];
}

// The trial intrinsics from the step d.
FID_HD void calib_lm_trial_intrinsics(CalibLM* s, const double d[9]) {
    for (int a = 0; a < 9; a++) {
        s->dint[a] = d[a];
        s->in[a] = s->in_prev[a] - d[a];
    }
    if (s->aspect != 0) s->in[0] = s->in[1] * s->aspect;
}

// CvLevMarq's (updateAlt) schedule after a trial of cost `err` from the J of cost `prev_err`, with the step's |p - pp|^2 = dn and
// |pp|^2 = pn: a trial whose cost exceeds prev_err raises lg and is retried from the same J while lg <= 16 (false, state stays 1);
// a kept trial lowers lg (>= -16), counts one iteration and sets state 2 after max_iter iterations or when
// |p - pp| / (|pp| + DBL_EPSILON) < eps, else 0 (true).  Shared by the calibrations and the map bundle adjustment (map_ba.cuh).
FID_HD bool lm_schedule_decide(int* state, int* lg, int* iters, int max_iter, double eps, double err, double prev_err, double dn, double pn) {
    const bool keep = !(err > prev_err && ++*lg <= 16);
    if (!keep) return false;
    *lg = *lg - 1 > -16 ? *lg - 1 : -16;
    ++*iters;
    *state = (*iters >= max_iter || sqrt(dn) / (sqrt(pn) + 2.220446049250313e-16) < eps) ? 2 : 0;
    return true;
}

// CvLevMarq's decision on a trial of cost `err` with the views' |p - pp|^2 and |pp|^2 summed in view order.
FID_HD void calib_lm_decide(CalibLM* s, double err, double dn_views, double pn_views) {
    double dn = 0.0, pn = 0.0;
    for (int a = 0; a < 9; a++) {
        dn += (s->in[a] - s->in_prev[a]) * (s->in[a] - s->in_prev[a]);
        pn += s->in_prev[a] * s->in_prev[a];
    }
    dn += dn_views;
    pn += pn_views;
    s->err = err;
    const bool keep = lm_schedule_decide(&s->state, &s->lg, &s->iters, s->max_iter, s->eps, err, s->prev_err, dn, pn);
    if (s->n_steps < CALIB_MAX_STEPS) s->steps[s->n_steps] = keep ? 1 : 0;
    s->n_steps++;
}

// Stage 5, one view: the standard deviations of its rvec and tvec given S^-1 (zero rows and columns for fixed intrinsics),
// from the undamped Schur block (scale 1).
FID_HD void calib_view_std(const double* blk, const double* sch, const double Sinv[9][9], double sigma2, double out[6]) {
    double Y[9][6], Z[9][6];
    for (int a = 0; a < 9; a++)
        for (int j = 0; j < 6; j++) {
            double s = 0.0;
            for (int k = 0; k < 6; k++) s += blk[CALIB_W + 6 * a + k] * sch[CALIB_VINV + 6 * k + j];
            Y[a][j] = s;
        }
    for (int a = 0; a < 9; a++)
        for (int j = 0; j < 6; j++) {
            double s = 0.0;
            for (int b = 0; b < 9; b++) s += Sinv[a][b] * Y[b][j];
            Z[a][j] = s;
        }
    for (int j = 0; j < 6; j++) {
        double s = sch[CALIB_VINV + 7 * j];
        for (int a = 0; a < 9; a++) s += Y[a][j] * Z[a][j];
        out[j] = sqrt(s * sigma2);
    }
}

// Stage 5: S^-1 of the undamped system (fixed rows and columns 0).
FID_HD void calib_schur_inverse(const double U[45], const double Q[45], const int mask[9], double Sinv[9][9]) {
    double S[9][9], r[9];
    const double zero[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    calib_schur_system(U, zero, Q, zero, 1.0, mask, S, r);
    for (int c = 0; c < 9; c++) {
        double u[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, x[9];
        u[c] = 1.0;
        solve_sym<9>(S, u, x);
        for (int a = 0; a < 9; a++) Sinv[a][c] = mask[a] && mask[c] ? x[a] : 0.0;
    }
}

// ---- object release: cv::calibrateCameraRO (calibrateCameraROExtended), DESIGN.md finding 21 ---------------------------------
// Every view holds the same n object points (the board); the parameters are the 9 intrinsics, 6 per view and the 3n board
// coordinates, of which the 7 of point 0, of point `fixed` and z of point n - 1 stay fixed.  J^T J gains the point blocks
// P_i = sum_v Jo^T Jo (3x3, a point enters only its own residuals), X_i = sum_v Ji^T Jo (9x3) and, per view, the cross columns
// Y_vi = Je^T Jo (6x3).  Eliminating the views' 6x6 blocks leaves the dense system over the m = 9 + 3n intrinsics and
// coordinates (fixed ones as identity rows): S = A - sum_v Z_v Z_v^T, Z_v = [W_v; Y_v] L_v^-T with L_v L_v^T the damped V_v,
// r = g - sum_v Z_v h_v, h_v = L_v^-1 ge_v; the dense kernels of calib_dense.cuh factor it (the host build: a plain Cholesky).
#define CALIB_PT_X 0   // per point: X 9x3 row-major 27
#define CALIB_PT_P 27  // P upper 6 (xx xy xz yy yz zz)
#define CALIB_PT_G 33  // go = sum Jo^T e 3
#define CALIB_PT 36
#define CALIB_FAC_L 0   // per view: L of the damped V, lower, packed row by row 21
#define CALIB_FAC_H 21  // h = L^-1 ge 6
#define CALIB_FAC 27
#define CALIB_RO_MAX_POINTS 1024  // per view: m <= 3081
#define CALIB_RO_MAX_VIEWS 4096

// d (u, v) / d (X, Y, Z) of one point from its d (u, v) / d t: the point enters the camera frame as R X + t.
FID_HD void calib_point_obj(const double Je[2][6], const double R[9], double Jo[2][3]) {
    for (int r = 0; r < 2; r++)
        for (int c = 0; c < 3; c++) Jo[r][c] = Je[r][3] * R[c] + Je[r][4] * R[3 + c] + Je[r][5] * R[6 + c];
}

// The release mask: coordinate c of point i is free unless it is one of point 0's, one of point `fixed`'s or z of point n - 1.
FID_HD bool calib_ro_free(int i, int c, int n, int fixed) { return i != 0 && i != fixed && !(i == n - 1 && c == 2); }

// Free parameters of a released run (the sigma^2 count): the free intrinsics, 6 per view and 3n - 7 coordinates.
FID_HD int calib_ro_nfree(const int mask[9], int nv, int n) {
    int k = 6 * nv + 3 * n - 7;
    for (int a = 0; a < 9; a++) k += mask[a];
    return k;
}

// Point i's sums over the views, in view order (layout CALIB_PT_*), at intrinsics `in`, the views' extrinsics p[6 nv] and the
// board obj[3n]; img holds n points per view.
FID_HD void calib_ro_point_sums(int nv, int n, int i, const double* obj, const float* img, const double in[9], double aspect, const double* p, double* out) {
    for (int k = 0; k < CALIB_PT; k++) out[k] = 0.0;
    for (int v = 0; v < nv; v++) {
        double R[9], dRdr[27], e[2], Ji[2][9], Je[2][6], Jo[2][3];
        rodrigues_v2m(p + 6 * v, R, dRdr);
        calib_point(obj + 3 * i, img + 2 * ((size_t)n * v + i), in, aspect, R, dRdr, p + 6 * v, e, Ji, Je);
        calib_point_obj(Je, R, Jo);
        for (int a = 0; a < 9; a++)
            for (int c = 0; c < 3; c++) out[CALIB_PT_X + 3 * a + c] += Ji[0][a] * Jo[0][c] + Ji[1][a] * Jo[1][c];
        for (int a = 0, o = 0; a < 3; a++)
            for (int b = a; b < 3; b++, o++) out[CALIB_PT_P + o] += Jo[0][a] * Jo[0][b] + Jo[1][a] * Jo[1][b];
        for (int c = 0; c < 3; c++) out[CALIB_PT_G + c] += Jo[0][c] * e[0] + Jo[1][c] * e[1];
    }
}

FID_HD void calib_ro_lsolve6(const double* L, const double b[6], double z[6]) {  // L z = b
    for (int a = 0; a < 6; a++) {
        double s = b[a];
        for (int k = 0; k < a; k++) s -= L[a * (a + 1) / 2 + k] * z[k];
        z[a] = s / L[a * (a + 1) / 2 + a];
    }
}
FID_HD void calib_ro_ltsolve6(const double* L, const double b[6], double x[6]) {  // L^T x = b
    for (int a = 5; a >= 0; a--) {
        double s = b[a];
        for (int k = a + 1; k < 6; k++) s -= L[k * (k + 1) / 2 + a] * x[k];
        x[a] = s / L[a * (a + 1) / 2 + a];
    }
}

// The Cholesky factor L (lower, packed row by row, 21) of the symmetric 6x6 matrix given by its upper triangle (21, row by row)
// with its diagonal times `scale`; false on a non-positive pivot.
FID_HD bool calib_chol6(const double* upper, double scale, double* L) {
    double A[6][6];
    for (int a = 0, o = 0; a < 6; a++)
        for (int b = a; b < 6; b++, o++) A[a][b] = A[b][a] = upper[o];
    for (int a = 0; a < 6; a++) A[a][a] *= scale;
    for (int a = 0; a < 6; a++)
        for (int b = 0; b <= a; b++) {
            double s = A[a][b];
            for (int k = 0; k < b; k++) s -= L[a * (a + 1) / 2 + k] * L[b * (b + 1) / 2 + k];
            if (a != b) {
                L[a * (a + 1) / 2 + b] = s / L[b * (b + 1) / 2 + b];
            } else {
                if (!(s > 0.0)) return false;
                L[a * (a + 1) / 2 + a] = sqrt(s);
            }
        }
    return true;
}

// One view: the Cholesky factor L of V with its diagonal times `scale`, and h = L^-1 ge (layout CALIB_FAC_*); false on a
// non-positive pivot.
FID_HD bool calib_ro_view_factor(const double* blk, double scale, double* fac) {
    if (!calib_chol6(blk + CALIB_V, scale, fac + CALIB_FAC_L)) return false;
    calib_ro_lsolve6(fac + CALIB_FAC_L, blk + CALIB_GE, fac + CALIB_FAC_H);
    return true;
}

// One view's 9 intrinsic rows of Z = W L^-T (rows of fixed intrinsics 0).
FID_HD void calib_ro_z_intrinsics(const double* blk, const double* fac, const int mask[9], double z[9][6]) {
    for (int a = 0; a < 9; a++) {
        const double zero[6] = {0, 0, 0, 0, 0, 0};
        calib_ro_lsolve6(fac + CALIB_FAC_L, mask[a] ? blk + CALIB_W + 6 * a : zero, z[a]);
    }
}

// One view's 3 rows of point i in Z = Y L^-T, Y = Je^T Jo of the point at `in`, p and the board coordinates o (rows of fixed
// coordinates 0).
FID_HD void calib_ro_z_point(const double* o, const float* m, const double in[9], double aspect, const double p[6], const double* fac, int i, int n, int fixed,
                             double z[3][6]) {
    double R[9], dRdr[27], e[2], Je[2][6], Jo[2][3];
    rodrigues_v2m(p, R, dRdr);
    calib_point(o, m, in, aspect, R, dRdr, p, e, nullptr, Je);
    calib_point_obj(Je, R, Jo);
    for (int c = 0; c < 3; c++) {
        double y[6];
        const bool f = calib_ro_free(i, c, n, fixed);
        for (int j = 0; j < 6; j++) y[j] = f ? Je[0][j] * Jo[0][c] + Je[1][j] * Jo[1][c] : 0.0;
        calib_ro_lsolve6(fac + CALIB_FAC_L, y, z[c]);
    }
}

// Entry (a, b), a >= b, of A = [U X; X^T P] (the diagonal times `scale`) over the m = 9 + 3n parameters; the rows and columns of
// fixed parameters, and the rows past m up to a padded size, are the identity.
FID_HD bool calib_ro_param_free(int a, int n, int fixed, const int mask[9]) {
    return a < 9 ? mask[a] != 0 : (a < 9 + 3 * n && calib_ro_free((a - 9) / 3, (a - 9) % 3, n, fixed));
}
FID_HD double calib_ro_entry(int a, int b, int n, int fixed, const int mask[9], const double U[45], const double* pts, double scale) {
    if (!calib_ro_param_free(a, n, fixed, mask) || !calib_ro_param_free(b, n, fixed, mask)) return a == b ? 1.0 : 0.0;
    double s;
    if (a < 9) {
        s = U[b * 9 - b * (b - 1) / 2 + a - b];
    } else if (b < 9) {
        s = pts[(size_t)CALIB_PT * ((a - 9) / 3) + CALIB_PT_X + 3 * b + (a - 9) % 3];
    } else {
        const int ia = (a - 9) / 3, ca = (a - 9) % 3, ib = (b - 9) / 3, cb = (b - 9) % 3;
        if (ia != ib) return 0.0;
        s = pts[(size_t)CALIB_PT * ia + CALIB_PT_P + cb * 3 - cb * (cb - 1) / 2 + ca - cb];
    }
    return a == b ? s * scale : s;
}
// Entry a of g = [gi; go] (0 for fixed parameters and past m).
FID_HD double calib_ro_grad(int a, int n, int fixed, const int mask[9], const double gi[9], const double* pts) {
    if (!calib_ro_param_free(a, n, fixed, mask)) return 0.0;
    return a < 9 ? gi[a] : pts[(size_t)CALIB_PT * ((a - 9) / 3) + CALIB_PT_G + (a - 9) % 3];
}

// Stage 4 with released points, one view: r = ge - W^T dint - sum_i Y_i dobj_i (Y at the J's parameters in_prev, pp, obj_prev),
// the step x = Vd^-1 r from the view's factor, p = pp - x and, at the trial parameters `in`, p and obj, out = {cost,
// |p - pp|^2, |pp|^2}.
FID_HD void calib_ro_view_trial(int n, const double* obj_prev, const double* obj, const double* dobj, const float* img, const double in_prev[9], const double in[9],
                                double aspect, const double* blk, const double* fac, const double dint[9], const double pp[6], double p[6], double out[3]) {
    double R[9], dRdr[27], t[6];
    rodrigues_v2m(pp, R, dRdr);
    board_sum<6>(n, [&](int i, double v[6]) {
        double e[2], Je[2][6], Jo[2][3];
        calib_point(obj_prev + 3 * i, img + 2 * i, in_prev, aspect, R, dRdr, pp, e, nullptr, Je);
        calib_point_obj(Je, R, Jo);
        const double* d = dobj + 3 * i;
        const double jd0 = Jo[0][0] * d[0] + Jo[0][1] * d[1] + Jo[0][2] * d[2], jd1 = Jo[1][0] * d[0] + Jo[1][1] * d[1] + Jo[1][2] * d[2];
        for (int k = 0; k < 6; k++) v[k] = Je[0][k] * jd0 + Je[1][k] * jd1;
    }, t);
    double r[6], z[6], x[6];
    for (int k = 0; k < 6; k++) {
        double s = blk[CALIB_GE + k];
        for (int a = 0; a < 9; a++) s -= blk[CALIB_W + 6 * a + k] * dint[a];
        r[k] = s - t[k];
    }
    calib_ro_lsolve6(fac + CALIB_FAC_L, r, z);
    calib_ro_ltsolve6(fac + CALIB_FAC_L, z, x);
    double dn = 0.0, pn = 0.0;
    for (int j = 0; j < 6; j++) {
        p[j] = pp[j] - x[j];
        dn += (p[j] - pp[j]) * (p[j] - pp[j]);
        pn += pp[j] * pp[j];
    }
    out[0] = calib_view_cost(n, obj, img, in, aspect, p);
    out[1] = dn;
    out[2] = pn;
}

// Stage 5 with released points, one view: the standard deviations of its rvec and tvec, diag(V^-1 + V^-1 B^T S^-1 B V^-1)
// sigma^2 from the undamped factor L (V = L L^T) and M = Z^T S^-1 Z (6x6, Z = B L^-T; M = T^T T with T = L_S^-1 Z).
FID_HD void calib_ro_view_std(const double* fac, const double M[36], double sigma2, double out[6]) {
    double Li[6][6];  // L^-1, column by column
    for (int c = 0; c < 6; c++) {
        double u[6] = {0, 0, 0, 0, 0, 0}, x[6];
        u[c] = 1.0;
        calib_ro_lsolve6(fac + CALIB_FAC_L, u, x);
        for (int r = 0; r < 6; r++) Li[r][c] = x[r];
    }
    for (int j = 0; j < 6; j++) {
        double s = 0.0;
        for (int k = 0; k < 6; k++) s += Li[k][j] * Li[k][j];
        for (int k = 0; k < 6; k++)
            for (int l = 0; l < 6; l++) s += Li[k][j] * M[6 * k + l] * Li[l][j];
        out[j] = sqrt(s * sigma2);
    }
}

// The step of the board coordinates: the trial board obj = obj_prev - d (d 0 for fixed coordinates), and |d|^2, |obj_prev|^2
// in coordinate order.
FID_HD void calib_ro_obj_trial(int n, int fixed, const double* obj_prev, const double* d, double* obj, double out[2]) {
    double dn = 0.0, pn = 0.0;
    for (int k = 0; k < 3 * n; k++) {
        const double dk = calib_ro_free(k / 3, k % 3, n, fixed) ? d[k] : 0.0;
        obj[k] = obj_prev[k] - dk;
        dn += (obj[k] - obj_prev[k]) * (obj[k] - obj_prev[k]);
        pn += obj_prev[k] * obj_prev[k];
    }
    out[0] = dn;
    out[1] = pn;
}

}  // namespace fid
