// Per-marker pose: cv::solvePnP(SOLVEPNP_ITERATIVE) on the 4 marker corners, as called by
// FiducialsNode::estimatePoseSingleMarkers (aruco_detect/src/aruco_detect.cpp:223-255, solvePnP at
// :247, object points :151-161), followed by getReprojectionError (:203-221), calcFiducialArea
// (:179-200) and the FiducialTransform packing of poseEstimateCallback (:447-495).
//
// solvePnP's planar branch restated from SURVEY.md A.9 / E.4 (validated there against cv2 on 335
// markers): undistort (5 fixed-point iterations) -> 4-point normalised-DLT homography (9x9
// symmetric eigenproblem) -> R from the orthonormalised homography columns -> Levenberg-Marquardt on
// the distorted reprojection error with OpenCV's CvLevMarq lambda schedule (max 20 iterations,
// eps FLT_EPSILON).  Everything is double; one marker per thread.
#pragma once
#include "common.cuh"

namespace fid {

// ---- small dense linear algebra ------------------------------------------------------------------
// Cyclic Jacobi eigen-decomposition of a symmetric NxN matrix: A = V diag(w) V^T (columns of V).
template <int N>
FID_HD void jacobi_eigen(double A[N][N], double w[N], double V[N][N]) {
    for (int i = 0; i < N; i++)
        for (int j = 0; j < N; j++) V[i][j] = i == j ? 1.0 : 0.0;
#pragma unroll 1
    for (int sweep = 0; sweep < 60; sweep++) {
        double off = 0.0, diag = 0.0;
        for (int i = 0; i < N; i++) {
            diag += A[i][i] * A[i][i];
            for (int j = i + 1; j < N; j++) off += A[i][j] * A[i][j];
        }
        if (off <= 1e-40 * diag || off == 0.0) break;
        // NOTE: keep the rotation loops rolled.  nvcc 12.9 (-O1..-O3) has miscompiled the fully unrolled
        // N=6 instance (eigenvalues wrong, off-diagonal mass not reduced; host build of the same source is
        // correct) -- found with tools/debug_pose.cu.
#pragma unroll 1
        for (int p = 0; p < N - 1; p++)
#pragma unroll 1
            for (int q = p + 1; q < N; q++) {
                const double apq = A[p][q];
                if (apq == 0.0) continue;
                const double theta = (A[q][q] - A[p][p]) / (2.0 * apq);
                const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
                for (int k = 0; k < N; k++) {
                    const double akp = A[k][p], akq = A[k][q];
                    A[k][p] = c * akp - s * akq;
                    A[k][q] = s * akp + c * akq;
                }
                for (int k = 0; k < N; k++) {
                    const double apk = A[p][k], aqk = A[q][k];
                    A[p][k] = c * apk - s * aqk;
                    A[q][k] = s * apk + c * aqk;
                }
                for (int k = 0; k < N; k++) {
                    const double vkp = V[k][p], vkq = V[k][q];
                    V[k][p] = c * vkp - s * vkq;
                    V[k][q] = s * vkp + c * vkq;
                }
            }
    }
    for (int i = 0; i < N; i++) w[i] = A[i][i];
}

FID_HD void mat3_mul(const double A[9], const double B[9], double C[9]) {
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) C[i * 3 + j] = A[i * 3] * B[j] + A[i * 3 + 1] * B[3 + j] + A[i * 3 + 2] * B[6 + j];
}

// Nearest orthogonal matrix (the U V^T of the SVD) by Newton iteration on the polar factor.
FID_HD void orthonormalize3(double R[9]) {
    for (int it = 0; it < 30; it++) {
        double T[9];
        // T = inverse-transpose of R
        const double c00 = R[4] * R[8] - R[5] * R[7], c01 = R[5] * R[6] - R[3] * R[8], c02 = R[3] * R[7] - R[4] * R[6];
        const double det = R[0] * c00 + R[1] * c01 + R[2] * c02;
        if (det == 0.0) return;
        const double id = 1.0 / det;
        T[0] = c00 * id;
        T[1] = c01 * id;
        T[2] = c02 * id;
        T[3] = (R[2] * R[7] - R[1] * R[8]) * id;
        T[4] = (R[0] * R[8] - R[2] * R[6]) * id;
        T[5] = (R[1] * R[6] - R[0] * R[7]) * id;
        T[6] = (R[1] * R[5] - R[2] * R[4]) * id;
        T[7] = (R[2] * R[3] - R[0] * R[5]) * id;
        T[8] = (R[0] * R[4] - R[1] * R[3]) * id;
        double delta = 0.0;
        for (int i = 0; i < 9; i++) {
            const double n = 0.5 * (R[i] + T[i]);
            delta += fabs(n - R[i]);
            R[i] = n;
        }
        if (delta < 1e-15) break;
    }
}

// cv::Rodrigues, matrix -> vector (orthonormalises first).
FID_HD void rodrigues_m2v(const double Rin[9], double r[3]) {
    double R[9];
    for (int i = 0; i < 9; i++) R[i] = Rin[i];
    orthonormalize3(R);
    double rx = R[7] - R[5], ry = R[2] - R[6], rz = R[3] - R[1];
    const double s = sqrt((rx * rx + ry * ry + rz * rz) * 0.25);
    double c = (R[0] + R[4] + R[8] - 1.0) * 0.5;
    c = c > 1.0 ? 1.0 : (c < -1.0 ? -1.0 : c);
    double theta = acos(c);
    if (s < 1e-5) {
        if (c > 0) {
            r[0] = r[1] = r[2] = 0.0;
            return;
        }
        double t = (R[0] + 1.0) * 0.5;
        rx = sqrt(t > 0.0 ? t : 0.0);
        t = (R[4] + 1.0) * 0.5;
        ry = sqrt(t > 0.0 ? t : 0.0) * (R[1] < 0 ? -1.0 : 1.0);
        t = (R[8] + 1.0) * 0.5;
        rz = sqrt(t > 0.0 ? t : 0.0) * (R[2] < 0 ? -1.0 : 1.0);
        if (fabs(rx) < fabs(ry) && fabs(rx) < fabs(rz) && ((R[5] > 0) != (ry * rz > 0))) rz = -rz;
        theta /= sqrt(rx * rx + ry * ry + rz * rz);
        r[0] = rx * theta;
        r[1] = ry * theta;
        r[2] = rz * theta;
        return;
    }
    const double vth = (1.0 / (2.0 * s)) * theta;
    r[0] = rx * vth;
    r[1] = ry * vth;
    r[2] = rz * vth;
}

// cv::Rodrigues, vector -> matrix, optionally with dR/dr (J[i*9+k] = d R[k] / d r_i).
FID_HD void rodrigues_v2m(const double r[3], double R[9], double* J) {
    const double theta = sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
    if (theta < 2.220446049250313e-16) {
        for (int i = 0; i < 9; i++) R[i] = (i % 4 == 0) ? 1.0 : 0.0;
        if (J) {
            for (int i = 0; i < 27; i++) J[i] = 0.0;
            J[5] = J[15] = J[19] = -1.0;
            J[7] = J[11] = J[21] = 1.0;
        }
        return;
    }
    const double c = cos(theta), s = sin(theta), c1 = 1.0 - c, itheta = 1.0 / theta;
    const double rx = r[0] * itheta, ry = r[1] * itheta, rz = r[2] * itheta;
    const double rrt[9] = {rx * rx, rx * ry, rx * rz, rx * ry, ry * ry, ry * rz, rx * rz, ry * rz, rz * rz};
    const double r_x[9] = {0, -rz, ry, rz, 0, -rx, -ry, rx, 0};
    for (int k = 0; k < 9; k++) R[k] = c * ((k % 4 == 0) ? 1.0 : 0.0) + c1 * rrt[k] + s * r_x[k];
    if (J) {
        const double drrt[27] = {rx + rx, ry, rz, ry, 0, 0, rz, 0, 0, 0, rx, 0, rx, ry + ry, rz, 0, rz, 0, 0, 0, rx, 0, 0, ry, rx, ry, rz + rz};
        const double d_r_x[27] = {0, 0, 0, 0, 0, -1, 0, 1, 0, 0, 0, 1, 0, 0, 0, -1, 0, 0, 0, -1, 0, 1, 0, 0, 0, 0, 0};
        for (int i = 0; i < 3; i++) {
            const double ri = i == 0 ? rx : (i == 1 ? ry : rz);
            const double a0 = -s * ri, a1 = (s - 2 * c1 * itheta) * ri, a2 = c1 * itheta;
            const double a3 = (c - s * itheta) * ri, a4 = s * itheta;
            for (int k = 0; k < 9; k++)
                J[i * 9 + k] = a0 * ((k % 4 == 0) ? 1.0 : 0.0) + a1 * rrt[k] + a2 * drrt[i * 9 + k] + a3 * r_x[k] + a4 * d_r_x[i * 9 + k];
        }
    }
}

struct Camera {
    double fx, fy, cx, cy;
    double k1, k2, p1, p2, k3;  // plumb_bob, first 5 coefficients (aruco_detect.cpp:317-323)
};

// cv::projectPoints for 4 object points; uv[8] = (u0,v0,...); Jm[8][6] = d(u,v)/d(r,t) if non-null.
FID_HD void project4(const double obj[4][3], const double p[6], const Camera& cam, double uv[8], double (*Jm)[6]) {
    double R[9], dRdr[27];
    rodrigues_v2m(p, R, Jm ? dRdr : nullptr);
    for (int i = 0; i < 4; i++) {
        const double X = obj[i][0], Y = obj[i][1], Z = obj[i][2];
        double x = R[0] * X + R[1] * Y + R[2] * Z + p[3];
        double y = R[3] * X + R[4] * Y + R[5] * Z + p[4];
        double z = R[6] * X + R[7] * Y + R[8] * Z + p[5];
        z = z != 0.0 ? 1.0 / z : 1.0;
        x *= z;
        y *= z;
        const double r2 = x * x + y * y, r4 = r2 * r2, r6 = r4 * r2;
        const double a1 = 2 * x * y, a2 = r2 + 2 * x * x, a3 = r2 + 2 * y * y;
        const double cdist = 1 + cam.k1 * r2 + cam.k2 * r4 + cam.k3 * r6;
        const double xd = x * cdist + cam.p1 * a1 + cam.p2 * a2;
        const double yd = y * cdist + cam.p1 * a3 + cam.p2 * a1;
        uv[2 * i] = xd * cam.fx + cam.cx;
        uv[2 * i + 1] = yd * cam.fy + cam.cy;
        if (Jm) {
            // translation part
            double dxd[6], dyd[6];  // d(x)/dparam, d(y)/dparam for the 6 parameters (r then t)
            for (int j = 0; j < 3; j++) {
                const double dx0 = X * dRdr[j * 9 + 0] + Y * dRdr[j * 9 + 1] + Z * dRdr[j * 9 + 2];
                const double dy0 = X * dRdr[j * 9 + 3] + Y * dRdr[j * 9 + 4] + Z * dRdr[j * 9 + 5];
                const double dz0 = X * dRdr[j * 9 + 6] + Y * dRdr[j * 9 + 7] + Z * dRdr[j * 9 + 8];
                dxd[j] = z * (dx0 - x * dz0);
                dyd[j] = z * (dy0 - y * dz0);
            }
            dxd[3] = z;
            dxd[4] = 0;
            dxd[5] = -x * z;
            dyd[3] = 0;
            dyd[4] = z;
            dyd[5] = -y * z;
            for (int j = 0; j < 6; j++) {
                const double dr2 = 2 * x * dxd[j] + 2 * y * dyd[j];
                const double dcdist = cam.k1 * dr2 + 2 * cam.k2 * r2 * dr2 + 3 * cam.k3 * r4 * dr2;
                const double da1 = 2 * (x * dyd[j] + y * dxd[j]);
                const double dmx = dxd[j] * cdist + x * dcdist + cam.p1 * da1 + cam.p2 * (dr2 + 4 * x * dxd[j]);
                const double dmy = dyd[j] * cdist + y * dcdist + cam.p1 * (dr2 + 4 * y * dyd[j]) + cam.p2 * da1;
                Jm[2 * i][j] = cam.fx * dmx;
                Jm[2 * i + 1][j] = cam.fy * dmy;
            }
        }
    }
}

// Gaussian elimination with partial pivoting, N x N, in place; returns false if singular.
template <int N>
FID_HD bool solve_linear(double A[N][N], double b[N]) {
#pragma unroll 1
    for (int i = 0; i < N; i++) {
        int k = i;
        for (int j = i + 1; j < N; j++)
            if (fabs(A[j][i]) > fabs(A[k][i])) k = j;
        if (fabs(A[k][i]) < 1e-300) return false;
        if (k != i) {
            for (int j = i; j < N; j++) {
                const double t = A[i][j];
                A[i][j] = A[k][j];
                A[k][j] = t;
            }
            const double t = b[i];
            b[i] = b[k];
            b[k] = t;
        }
        const double d = 1.0 / A[i][i];
        for (int j = i + 1; j < N; j++) {
            const double alpha = A[j][i] * d;
            for (int c = i + 1; c < N; c++) A[j][c] -= alpha * A[i][c];
            b[j] -= alpha * b[i];
        }
    }
#pragma unroll 1
    for (int i = N - 1; i >= 0; i--) {
        double s = b[i];
        for (int c = i + 1; c < N; c++) s -= A[i][c] * b[c];
        b[i] = s / A[i][i];
    }
    return true;
}

// 4-point homography src(x,y) -> dst(x,y).  OpenCV takes the eigenvector of the smallest eigenvalue
// of the normalised 9x9 DLT matrix L^T L; for exactly 4 correspondences that null vector is the
// exact solution of the 8 DLT equations, so it is obtained here by solving them directly (in the same
// normalised coordinates, h22 = 1) -- identical up to rounding (~1e-14), far cheaper than a 9x9
// Jacobi sweep.  If the normalised h22 vanishes (degenerate view) fall back to the eigenvector.
FID_HD void homography4(const double src[4][2], const double dst[4][2], double Hm[9]) {
    double cm[2] = {0, 0}, cM[2] = {0, 0}, sm[2] = {0, 0}, sM[2] = {0, 0};
    for (int i = 0; i < 4; i++) {
        cm[0] += dst[i][0];
        cm[1] += dst[i][1];
        cM[0] += src[i][0];
        cM[1] += src[i][1];
    }
    for (int k = 0; k < 2; k++) {
        cm[k] /= 4;
        cM[k] /= 4;
    }
    for (int i = 0; i < 4; i++) {
        sm[0] += fabs(dst[i][0] - cm[0]);
        sm[1] += fabs(dst[i][1] - cm[1]);
        sM[0] += fabs(src[i][0] - cM[0]);
        sM[1] += fabs(src[i][1] - cM[1]);
    }
    for (int k = 0; k < 2; k++) {
        sm[k] = 4 / sm[k];
        sM[k] = 4 / sM[k];
    }
    double H0[9];
    double A[8][8], bb[8];
    for (int i = 0; i < 4; i++) {
        const double x = (dst[i][0] - cm[0]) * sm[0], y = (dst[i][1] - cm[1]) * sm[1];
        const double X = (src[i][0] - cM[0]) * sM[0], Y = (src[i][1] - cM[1]) * sM[1];
        const double r0[8] = {X, Y, 1, 0, 0, 0, -x * X, -x * Y};
        const double r1[8] = {0, 0, 0, X, Y, 1, -y * X, -y * Y};
        for (int k = 0; k < 8; k++) {
            A[2 * i][k] = r0[k];
            A[2 * i + 1][k] = r1[k];
        }
        bb[2 * i] = x;
        bb[2 * i + 1] = y;
    }
    bool ok = solve_linear<8>(A, bb);
    if (ok) {
        for (int k = 0; k < 8; k++) {
            H0[k] = bb[k];
            if (!(fabs(bb[k]) < 1e12)) ok = false;
        }
        H0[8] = 1.0;
    }
    if (!ok) {
        double LtL[9][9];
        for (int i = 0; i < 9; i++)
            for (int j = 0; j < 9; j++) LtL[i][j] = 0.0;
        for (int i = 0; i < 4; i++) {
            const double x = (dst[i][0] - cm[0]) * sm[0], y = (dst[i][1] - cm[1]) * sm[1];
            const double X = (src[i][0] - cM[0]) * sM[0], Y = (src[i][1] - cM[1]) * sM[1];
            const double Lx[9] = {X, Y, 1, 0, 0, 0, -x * X, -x * Y, -x};
            const double Ly[9] = {0, 0, 0, X, Y, 1, -y * X, -y * Y, -y};
            for (int j = 0; j < 9; j++)
                for (int k = 0; k < 9; k++) LtL[j][k] += Lx[j] * Lx[k] + Ly[j] * Ly[k];
        }
        double w[9], V[9][9];
        jacobi_eigen<9>(LtL, w, V);
        int best = 0;
        for (int i = 1; i < 9; i++)
            if (w[i] < w[best]) best = i;
        for (int i = 0; i < 9; i++) H0[i] = V[i][best];
    }
    const double invHnorm[9] = {1.0 / sm[0], 0, cm[0], 0, 1.0 / sm[1], cm[1], 0, 0, 1};
    const double Hnorm2[9] = {sM[0], 0, -cM[0] * sM[0], 0, sM[1], -cM[1] * sM[1], 0, 0, 1};
    double T[9];
    mat3_mul(invHnorm, H0, T);
    mat3_mul(T, Hnorm2, Hm);
    const double inv = 1.0 / Hm[8];
    for (int i = 0; i < 9; i++) Hm[i] *= inv;
}

// Solve the LM normal equations A x = b (A symmetric; positive definite after the (1+lambda) diagonal
// scaling).  OpenCV uses cv::solve(DECOMP_SVD); for a positive definite system the solutions agree
// to rounding, so a pivoted elimination is used and the eigen-decomposition (with DECOMP_SVD's
// singular-value cut-off) is kept only for the rank-deficient case.
// Out of line on the device: inlined into k_pose, nvcc 12.9 (sm_90a, NVVM -O3) miscompiles it -- the LM step comes out
// wrong and the solver stops after one iteration, rvec off by ~5e-3 (the same source inlined elsewhere, built with
// -Xcicc -O1, or called out of line gives the host result to 1e-14).
#if defined(__CUDACC__)
__host__ __device__ __noinline__
#else
inline
#endif
void solve_sym6(const double Ain[6][6], const double b[6], double x[6]) {
    double A[6][6];
    for (int i = 0; i < 6; i++) {
        x[i] = b[i];
        for (int j = 0; j < 6; j++) A[i][j] = Ain[i][j];
    }
    // conditioning guard: smallest pivot relative to the largest diagonal entry
    double dmax = 0.0;
    for (int i = 0; i < 6; i++) dmax = fabs(Ain[i][i]) > dmax ? fabs(Ain[i][i]) : dmax;
    bool ok = solve_linear<6>(A, x);
    if (ok) {
        for (int i = 0; i < 6; i++)
            if (!(fabs(A[i][i]) > 1e-11 * dmax)) ok = false;  // A now holds U; tiny pivot => near singular
    }
    if (ok) return;
    double w[6], V[6][6];
    for (int i = 0; i < 6; i++)
        for (int j = 0; j < 6; j++) A[i][j] = Ain[i][j];
    jacobi_eigen<6>(A, w, V);
    double thr = 0.0;
    for (int i = 0; i < 6; i++) thr += fabs(w[i]);
    thr *= 2.220446049250313e-16 * 2;
    for (int i = 0; i < 6; i++) x[i] = 0.0;
    for (int k = 0; k < 6; k++) {
        if (fabs(w[k]) <= thr) continue;
        double s = 0.0;
        for (int i = 0; i < 6; i++) s += V[i][k] * b[i];
        s /= w[k];
        for (int i = 0; i < 6; i++) x[i] += s * V[i][k];
    }
}

struct PoseOut {
    double rvec[3], tvec[3];
    double image_error, object_error, area;
    double quat[4];  // x y z w
    int lm_iters;
};

FID_HD double dist2f(float x1, float y1, float x2, float y2) {
    const double dx = (double)x1 - (double)x2, dy = (double)y1 - (double)y2;
    return sqrt(dx * dx + dy * dy);
}

// corners: 4 x (x,y) float32 in marker order TL,TR,BR,BL.  marker_len_f: this marker's side (already
// narrowed to float, :151), default_len: fiducial_len used for object_error (:493-495).
FID_HD void solve_marker_pose(const float corners[8], const Camera& cam, float marker_len_f, double default_len, PoseOut* out) {
    const float hf = marker_len_f / 2.f;
    const double h = hf;
    const double obj[4][3] = {{-h, h, 0}, {h, h, 0}, {h, -h, 0}, {-h, -h, 0}};
    double img[8];
    for (int i = 0; i < 8; i++) img[i] = corners[i];
    // 1. normalise + undistort
    double mn[4][2];
    for (int i = 0; i < 4; i++) {
        const double x0 = (img[2 * i] - cam.cx) / cam.fx, y0 = (img[2 * i + 1] - cam.cy) / cam.fy;
        double x = x0, y = y0;
        for (int it = 0; it < 5; it++) {
            const double r2 = x * x + y * y;
            const double icd = 1.0 / (1 + ((cam.k3 * r2 + cam.k2) * r2 + cam.k1) * r2);
            const double dx = 2 * cam.p1 * x * y + cam.p2 * (r2 + 2 * x * x);
            const double dy = cam.p1 * (r2 + 2 * y * y) + 2 * cam.p2 * x * y;
            x = (x0 - dx) * icd;
            y = (y0 - dy) * icd;
        }
        mn[i][0] = x;
        mn[i][1] = y;
    }
    // 2-4. planar initialisation (object plane is z=0 with zero centroid => Rt = I, Tt = 0)
    double src[4][2];
    for (int i = 0; i < 4; i++) {
        src[i][0] = obj[i][0];
        src[i][1] = obj[i][1];
    }
    double Hm[9];
    homography4(src, mn, Hm);
    double h1[3] = {Hm[0], Hm[3], Hm[6]}, h2[3] = {Hm[1], Hm[4], Hm[7]}, h3[3] = {Hm[2], Hm[5], Hm[8]};
    const double n1 = sqrt(h1[0] * h1[0] + h1[1] * h1[1] + h1[2] * h1[2]);
    const double n2 = sqrt(h2[0] * h2[0] + h2[1] * h2[1] + h2[2] * h2[2]);
    const double eps = 2.220446049250313e-16;
    const double d1 = 1.0 / (n1 > eps ? n1 : eps), d2 = 1.0 / (n2 > eps ? n2 : eps);
    const double d3 = 2.0 / ((n1 + n2) > eps ? (n1 + n2) : eps);
    for (int k = 0; k < 3; k++) {
        h1[k] *= d1;
        h2[k] *= d2;
        h3[k] *= d3;
    }
    const double t0[3] = {h3[0], h3[1], h3[2]};
    const double hx[3] = {h1[1] * h2[2] - h1[2] * h2[1], h1[2] * h2[0] - h1[0] * h2[2], h1[0] * h2[1] - h1[1] * h2[0]};
    double Rh[9] = {h1[0], h2[0], hx[0], h1[1], h2[1], hx[1], h1[2], h2[2], hx[2]};
    double p[6];
    rodrigues_m2v(Rh, p);
    // (cv converts rvec -> R -> rvec again; the second conversion is the identity up to rounding)
    double Rm[9];
    rodrigues_v2m(p, Rm, nullptr);
    rodrigues_m2v(Rm, p);
    p[3] = t0[0];
    p[4] = t0[1];
    p[5] = t0[2];
#ifdef FID_DEBUG_PNP
    printf("H %.17g %.17g %.17g %.17g %.17g %.17g %.17g %.17g\n", Hm[0], Hm[1], Hm[2], Hm[3], Hm[4], Hm[5], Hm[6], Hm[7]);
    printf("init %.17g %.17g %.17g %.17g %.17g %.17g\n", p[0], p[1], p[2], p[3], p[4], p[5]);
#endif
    // 5. Levenberg-Marquardt (CvLevMarq schedule)
    double uv[8], J[8][6], err[8];
    project4(obj, p, cam, uv, J);
    for (int i = 0; i < 8; i++) err[i] = uv[i] - img[i];
    int lam = -3, iters = 0;
    double prev_err = 0.0, en = 0.0;
    for (;;) {
        double JtJ[6][6], JtE[6], prev[6];
        for (int a = 0; a < 6; a++) {
            JtE[a] = 0.0;
            for (int k = 0; k < 8; k++) JtE[a] += J[k][a] * err[k];
            for (int b = 0; b < 6; b++) {
                double s = 0.0;
                for (int k = 0; k < 8; k++) s += J[k][a] * J[k][b];
                JtJ[a][b] = s;
            }
            prev[a] = p[a];
        }
        if (iters == 0) {
            double s = 0.0;
            for (int i = 0; i < 8; i++) s += err[i] * err[i];
            prev_err = sqrt(s);
        }
        for (;;) {
            double A[6][6], delta[6];
            const double scale = 1.0 + exp(lam * 2.302585092994046);
            for (int a = 0; a < 6; a++)
                for (int b = 0; b < 6; b++) A[a][b] = a == b ? JtJ[a][b] * scale : JtJ[a][b];
            solve_sym6(A, JtE, delta);
#ifdef FID_DEBUG_PNP
            if (iters == 0) {
                printf("J0 %.17g %.17g %.17g %.17g %.17g %.17g\n", J[0][0], J[0][1], J[0][2], J[0][3], J[0][4], J[0][5]);
                printf("J7 %.17g %.17g %.17g %.17g %.17g %.17g\n", J[7][0], J[7][1], J[7][2], J[7][3], J[7][4], J[7][5]);
                printf("JtE %.17g %.17g %.17g %.17g %.17g %.17g\n", JtE[0], JtE[1], JtE[2], JtE[3], JtE[4], JtE[5]);
                printf("Adiag %.17g %.17g %.17g %.17g %.17g %.17g scale %.17g\n", A[0][0], A[1][1], A[2][2], A[3][3], A[4][4], A[5][5], scale);
                printf("delta %.17g %.17g %.17g %.17g %.17g %.17g\n", delta[0], delta[1], delta[2], delta[3], delta[4], delta[5]);
            }
#endif
            for (int a = 0; a < 6; a++) p[a] = prev[a] - delta[a];
            project4(obj, p, cam, uv, nullptr);
            double s = 0.0;
            for (int i = 0; i < 8; i++) {
                const double e = uv[i] - img[i];
                s += e * e;
            }
            en = sqrt(s);
            if (en > prev_err) {
                lam++;
                if (lam <= 16) continue;
            }
            break;
        }
        lam = lam - 1 > -16 ? lam - 1 : -16;
        iters++;
#ifdef FID_DEBUG_PNP
        printf("it %d lam %d en %.17g prev %.17g p %.17g %.17g %.17g\n", iters, lam, en, prev_err, p[0], p[1], p[2]);
#endif
        double dn = 0.0, pn = 0.0;
        for (int a = 0; a < 6; a++) {
            dn += (p[a] - prev[a]) * (p[a] - prev[a]);
            pn += prev[a] * prev[a];
        }
        if (iters >= 20 || sqrt(dn) / sqrt(pn) < 1.1920928955078125e-07) break;
        prev_err = en;
        project4(obj, p, cam, uv, J);
        for (int i = 0; i < 8; i++) err[i] = uv[i] - img[i];
    }
    out->lm_iters = iters;
    for (int k = 0; k < 3; k++) {
        out->rvec[k] = p[k];
        out->tvec[k] = p[3 + k];
    }
    // 6. glue: reprojection error with the projected points rounded to float32 (:208-219)
    project4(obj, p, cam, uv, nullptr);
    double total = 0.0;
    for (int i = 0; i < 4; i++) {
        const double e = dist2f(corners[2 * i], corners[2 * i + 1], (float)uv[2 * i], (float)uv[2 * i + 1]);
        total += e * e;
    }
    out->image_error = total / 4.0;
    // calcFiducialArea (:179-200)
    {
        const float* c = corners;
        double a1 = dist2f(c[0], c[1], c[2], c[3]), b1 = dist2f(c[0], c[1], c[6], c[7]), c1 = dist2f(c[2], c[3], c[6], c[7]);
        double a2 = dist2f(c[2], c[3], c[4], c[5]), b2 = dist2f(c[4], c[5], c[6], c[7]), c2 = c1;
        const double s1 = (a1 + b1 + c1) / 2.0, s2 = (a2 + b2 + c2) / 2.0;
        a1 = sqrt(s1 * (s1 - a1) * (s1 - b1) * (s1 - c1));
        a2 = sqrt(s2 * (s2 - a2) * (s2 - b2) * (s2 - c2));
        out->area = a1 + a2;
    }
    // quaternion (:447-448, :485) and object_error (:493-495)
    const double angle = sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]);
    const double ax = p[0] / angle, ay = p[1] / angle, az = p[2] / angle;
    const double dlen = sqrt(ax * ax + ay * ay + az * az);
    const double s = sin(angle * 0.5) / dlen;
    out->quat[0] = ax * s;
    out->quat[1] = ay * s;
    out->quat[2] = az * s;
    out->quat[3] = cos(angle * 0.5);
    const double tn = sqrt(p[3] * p[3] + p[4] * p[4] + p[5] * p[5]);
    out->object_error = (out->image_error / dist2f(corners[0], corners[1], corners[4], corners[5])) * (tn / default_len);
}

}  // namespace fid
