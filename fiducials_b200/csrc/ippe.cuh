// Both planar pose hypotheses of one square marker: cv::solvePnPGeneric(obj, corners, K, D, flags=SOLVEPNP_IPPE_SQUARE)
// of OpenCV 4.13 (calib3d solvepnp.cpp + IPPE::PoseSolver::solveSquare, ippe.cpp; Collins & Bartoli, "Infinitesimal Plane-based
// Pose Estimation", IJCV 2014), with the object points of solve_marker_pose (the side narrowed to float, TL, TR, BR, BL -- the
// order SOLVEPNP_IPPE_SQUARE requires).  The published pose stays the ITERATIVE one of pnp.cuh; this only reports the two
// solutions a square admits, ordered and with their reprojection RMS, and which of them the ITERATIVE pose lies in.
//
//   1. undistort the corners to normalised coordinates (cv::undistortPoints, default criteria: the 5 fixed-point iterations of
//      pnp.cuh step 1).  undistortPoints returns float32 for float32 input, so the normalised points are rounded to float.
//   2. analytic homography of the square [-h,h]^2 onto them (homographyFromSquarePoints); |det| < 1e-9 -> no solution.
//   3. IPPE canonical form: Jacobian of the homography at the marker centre -> the two rotations (computeRotations), the
//      least-squares translation of each (computeTranslation).
//   4. order: the solver's own reprojection error in normalised coordinates, float arithmetic (evalReprojError); solvePnPGeneric
//      puts solution a first iff err_a < err_b (a tie puts b first).
//   5. per solution the RMS solvePnPGeneric reports: projectPoints with K and D, norm / sqrt(2n).
// All double, one marker per thread.
#pragma once
#include "pnp.cuh"

namespace fid {

struct PoseHypOut {
    int n;                  // 2, or 0 when IPPE has no solution (degenerate quad)
    int iterative_match;    // index of the solution whose rotation is closer to the ITERATIVE pose; -1 when n == 0
    double rvec[2][3], tvec[2][3];
    double rms[2];          // px, solvePnPGeneric's order
    float solver_err[2];    // the errors that decide the order (normalised coordinates)
};

// IPPE::PoseSolver::rotateVec2ZAxis, transposed: the rotation that takes the z axis to the direction of (p, q, 1).
FID_HD void ippe_rv(double p, double q, double Rv[9]) {
    const double nrm = sqrt(p * p + q * q + 1.0);
    const double ax = p / nrm, ay = q / nrm, c = 1.0 / nrm;
    const double d = 1.0 / (1.0 + c);  // c > 0: never the antipodal case
    const double ax2 = ax * ax, ay2 = ay * ay, axay = ax * ay;
    Rv[0] = -ax2 * d + 1.0;
    Rv[1] = -axay * d;
    Rv[2] = ax;
    Rv[3] = -axay * d;
    Rv[4] = -ay2 * d + 1.0;
    Rv[5] = ay;
    Rv[6] = -ax;
    Rv[7] = -ay;
    Rv[8] = 1.0 - (ax2 + ay2) * d;
}

// IPPE::PoseSolver::computeTranslation: least-squares t of R X + t ~ (u, v, 1) over the four points (normal equations).
FID_HD void ippe_translation(const double obj[4][3], const double un[4][2], const double R[9], double t[3]) {
    double A02 = 0, A12 = 0, A22 = 0, b0 = 0, b1 = 0, b2 = 0;
    const double A00 = 4.0, A11 = 4.0;
    for (int i = 0; i < 4; i++) {
        const double rx = R[0] * obj[i][0] + R[1] * obj[i][1];
        const double ry = R[3] * obj[i][0] + R[4] * obj[i][1];
        const double rz = R[6] * obj[i][0] + R[7] * obj[i][1];
        const double a2 = -un[i][0], c2 = -un[i][1];
        A02 += a2;
        A12 += c2;
        A22 += a2 * a2 + c2 * c2;
        const double bx = -a2 * rz - rx, by = -c2 * rz - ry;
        b0 += bx;
        b1 += by;
        b2 += a2 * bx + c2 * by;
    }
    const double A20 = A02, A21 = A12;
    const double det_inv = 1.0 / (A00 * A11 * A22 - A00 * A12 * A21 - A02 * A11 * A20);
    const double S00 = A11 * A22 - A12 * A21, S01 = A02 * A21, S02 = -A02 * A11;
    const double S10 = A12 * A20, S11 = A00 * A22 - A02 * A20, S12 = -A00 * A12;
    const double S20 = -A11 * A20, S21 = -A00 * A21, S22 = A00 * A11;
    t[0] = det_inv * (S00 * b0 + S01 * b1 + S02 * b2);
    t[1] = det_inv * (S10 * b0 + S11 * b1 + S12 * b2);
    t[2] = det_inv * (S20 * b0 + S21 * b1 + S22 * b2);
}

// IPPE::PoseSolver::evalReprojError: projectPoints with K = I and no distortion.  The object points are float32, so the projected
// points come back as float; the squared differences are summed in float.
FID_HD float ippe_solver_err(const double obj[4][3], const double un[4][2], const double rvec[3], const double t[3]) {
    const Camera unit = {1.0, 1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    const double p[6] = {rvec[0], rvec[1], rvec[2], t[0], t[1], t[2]};
    double uv[8];
    project4(obj, p, unit, uv, nullptr);
    float e = 0.f;
    for (int i = 0; i < 4; i++) {
        const float dx = (float)uv[2 * i] - (float)un[i][0];
        const float dy = (float)uv[2 * i + 1] - (float)un[i][1];
        e += dx * dx + dy * dy;
    }
    return (float)sqrt((double)(e / 8.0f));
}

// corners: 4 x (x,y) float32, TL,TR,BR,BL.  marker_len_f: the marker's side narrowed to float (solve_marker_pose).  iter_rvec: the
// marker's SOLVEPNP_ITERATIVE rvec (fid_transform::rvec), for iterative_match.
FID_HD void solve_marker_hypotheses(const float corners[8], const Camera& cam, float marker_len_f, const double iter_rvec[3], PoseHypOut* out) {
    out->n = 0;
    out->iterative_match = -1;
    for (int s = 0; s < 2; s++) {
        for (int k = 0; k < 3; k++) out->rvec[s][k] = out->tvec[s][k] = 0.0;
        out->rms[s] = 0.0;
        out->solver_err[s] = 0.f;
    }
    const float hf = marker_len_f / 2.f;
    const double h = hf;
    const double obj[4][3] = {{-h, h, 0}, {h, h, 0}, {h, -h, 0}, {-h, -h, 0}};
    // 1. cv::undistortPoints (same iteration as solve_marker_pose), output rounded to float32
    double un[4][2];
    for (int i = 0; i < 4; i++) {
        const double x0 = ((double)corners[2 * i] - cam.cx) / cam.fx, y0 = ((double)corners[2 * i + 1] - cam.cy) / cam.fy;
        double x = x0, y = y0;
        for (int it = 0; it < 5; it++) {
            const double r2 = x * x + y * y;
            const double icd = 1.0 / (1 + ((cam.k3 * r2 + cam.k2) * r2 + cam.k1) * r2);
            const double dx = 2 * cam.p1 * x * y + cam.p2 * (r2 + 2 * x * x);
            const double dy = cam.p1 * (r2 + 2 * y * y) + 2 * cam.p2 * x * y;
            x = (x0 - dx) * icd;
            y = (y0 - dy) * icd;
        }
        un[i][0] = (float)x;
        un[i][1] = (float)y;
    }
    // 2. homography of the square (+-h) onto the normalised corners, H22 = 1 (homographyFromSquarePoints)
    const double p1x = -un[0][0], p1y = -un[0][1], p2x = -un[1][0], p2y = -un[1][1];
    const double p3x = -un[2][0], p3y = -un[2][1], p4x = -un[3][0], p4y = -un[3][1];
    const double det = h * (p1x * p2y - p2x * p1y - p1x * p4y + p2x * p3y - p3x * p2y + p4x * p1y + p3x * p4y - p4x * p3y);
    if (!(fabs(det) >= 1e-9)) return;  // OpenCV throws "Determinant is zero!"; solvePnPGeneric returns no solution
    const double di = -1.0 / det;
    const double H00 = di * (p1x * p3x * p2y - p2x * p3x * p1y - p1x * p4x * p2y + p2x * p4x * p1y - p1x * p3x * p4y + p1x * p4x * p3y + p2x * p3x * p4y - p2x * p4x * p3y);
    const double H01 = di * (p1x * p2x * p3y - p1x * p3x * p2y - p1x * p2x * p4y + p2x * p4x * p1y + p1x * p3x * p4y - p3x * p4x * p1y - p2x * p4x * p3y + p3x * p4x * p2y);
    const double H02 = di * h * (p1x * p2x * p3y - p2x * p3x * p1y - p1x * p2x * p4y + p1x * p4x * p2y - p1x * p4x * p3y + p3x * p4x * p1y + p2x * p3x * p4y - p3x * p4x * p2y);
    const double H10 = di * (p1x * p2y * p3y - p2x * p1y * p3y - p1x * p2y * p4y + p2x * p1y * p4y - p3x * p1y * p4y + p4x * p1y * p3y + p3x * p2y * p4y - p4x * p2y * p3y);
    const double H11 = di * (p2x * p1y * p3y - p3x * p1y * p2y - p1x * p2y * p4y + p4x * p1y * p2y + p1x * p3y * p4y - p4x * p1y * p3y - p2x * p3y * p4y + p3x * p2y * p4y);
    const double H12 = di * h * (p1x * p2y * p3y - p3x * p1y * p2y - p2x * p1y * p4y + p4x * p1y * p2y - p1x * p3y * p4y + p3x * p1y * p4y + p2x * p3y * p4y - p4x * p2y * p3y);
    const double H20 = -di * (p1x * p3y - p3x * p1y - p1x * p4y - p2x * p3y + p3x * p2y + p4x * p1y + p2x * p4y - p4x * p2y);
    const double H21 = di * (p1x * p2y - p2x * p1y - p1x * p3y + p3x * p1y + p2x * p4y - p4x * p2y - p3x * p4y + p4x * p3y);
    // 3. canonical form (solveCanonicalForm): Jacobian of H at the centre and the image (v0, v1) of the centre
    const double j00 = H00 - H20 * H02, j01 = H01 - H21 * H02, j10 = H10 - H20 * H12, j11 = H11 - H21 * H12;
    const double v0 = H02, v1 = H12;
    double Rv[9];
    ippe_rv(v0, v1, Rv);
    // computeRotations: the 2x2 block A = B^-1 J, its largest singular value gamma, the two completions of A / gamma
    const double b00 = Rv[0] - v0 * Rv[6], b01 = Rv[1] - v0 * Rv[7], b10 = Rv[3] - v1 * Rv[6], b11 = Rv[4] - v1 * Rv[7];
    const double dtinv = 1.0 / (b00 * b11 - b01 * b10);
    const double bi00 = dtinv * b11, bi01 = -dtinv * b01, bi10 = -dtinv * b10, bi11 = dtinv * b00;
    const double a00 = bi00 * j00 + bi01 * j10, a01 = bi00 * j01 + bi01 * j11;
    const double a10 = bi10 * j00 + bi11 * j10, a11 = bi10 * j01 + bi11 * j11;
    const double ata00 = a00 * a00 + a01 * a01, ata01 = a00 * a10 + a01 * a11, ata11 = a10 * a10 + a11 * a11;
    const double gamma2 = 0.5 * (ata00 + ata11 + sqrt((ata00 - ata11) * (ata00 - ata11) + 4.0 * ata01 * ata01));
    if (!(gamma2 >= 0.0)) return;  // "gamma2 is negative."
    const double gamma = sqrt(gamma2);
    if (!(gamma >= 1.1920928955078125e-07)) return;  // "gamma is zero."
    const double r00 = a00 / gamma, r01 = a01 / gamma, r10 = a10 / gamma, r11 = a11 / gamma;
    // 1 - |column|^2 is >= 0 in exact arithmetic (gamma is the largest singular value); clamp the rounding (OpenCV would give NaN)
    const double q0 = -r00 * r00 - r10 * r10 + 1.0, q1 = -r01 * r01 - r11 * r11 + 1.0;
    const double c0 = sqrt(q0 > 0.0 ? q0 : 0.0);
    double c1 = sqrt(q1 > 0.0 ? q1 : 0.0);
    if (-r00 * r01 - r10 * r11 < 0) c1 = -c1;
    double R[2][9];
    for (int s = 0; s < 2; s++) {
        const double e0 = s == 0 ? c0 : -c0, e1 = s == 0 ? c1 : -c1;
        const double m02 = e1 * r10 - e0 * r11, m12 = e0 * r01 - e1 * r00, m22 = r00 * r11 - r01 * r10;
        for (int i = 0; i < 3; i++) {  // R = Rv * [[r00 r01 m02] [r10 r11 m12] [e0 e1 m22]]
            const double w0 = Rv[3 * i], w1 = Rv[3 * i + 1], w2 = Rv[3 * i + 2];
            R[s][3 * i] = r00 * w0 + r10 * w1 + e0 * w2;
            R[s][3 * i + 1] = r01 * w0 + r11 * w1 + e1 * w2;
            R[s][3 * i + 2] = m02 * w0 + m12 * w1 + m22 * w2;
        }
    }
    double rv[2][3], tv[2][3];
    float err[2];
    for (int s = 0; s < 2; s++) {
        ippe_translation(obj, un, R[s], tv[s]);
        rodrigues_m2v(R[s], rv[s]);
        err[s] = ippe_solver_err(obj, un, rv[s], tv[s]);
    }
    // 4. order (sortPosesByReprojError, then solvePnPGeneric's `reprojErr1 < reprojErr2`)
    const int first = err[0] < err[1] ? 0 : 1;
    double Rit[9];
    rodrigues_v2m(iter_rvec, Rit, nullptr);
    double closeness[2];
    bool finite = true;
    for (int k = 0; k < 2; k++) {
        const int s = k == 0 ? first : 1 - first;
        const double p[6] = {rv[s][0], rv[s][1], rv[s][2], tv[s][0], tv[s][1], tv[s][2]};
        // 5. the RMS solvePnPGeneric reports: projectPoints with the camera's K and D against the given corners
        double uv[8], sq = 0.0;
        project4(obj, p, cam, uv, nullptr);
        for (int i = 0; i < 8; i++) {
            const double e = uv[i] - (double)corners[i];
            sq += e * e;
        }
        out->rms[k] = sqrt(sq) / sqrt(8.0);
        out->solver_err[k] = err[s];
        // iterative_match: trace(R_s^T R_iter) grows as the angle between the two rotations shrinks
        double tr = 0.0;
        for (int i = 0; i < 9; i++) tr += R[s][i] * Rit[i];
        closeness[k] = tr;
        for (int j = 0; j < 3; j++) {
            out->rvec[k][j] = rv[s][j];
            out->tvec[k][j] = tv[s][j];
            finite = finite && isfinite(rv[s][j]) && isfinite(tv[s][j]);
        }
        finite = finite && isfinite(out->rms[k]);
    }
    if (!finite) {  // only for inputs at the edge of the degenerate test; report no solution rather than NaN
        for (int s = 0; s < 2; s++) {
            for (int k = 0; k < 3; k++) out->rvec[s][k] = out->tvec[s][k] = 0.0;
            out->rms[s] = 0.0;
            out->solver_err[s] = 0.f;
        }
        return;
    }
    out->n = 2;
    out->iterative_match = closeness[1] > closeness[0] ? 1 : 0;
}

}  // namespace fid
