// CPU harness for the object-release part of fiducials_b200/csrc/calib.cuh (cv::calibrateCameraROExtended).  TEST INFRASTRUCTURE
// ONLY.  Compiled with g++ by tests/calib_ro_cases.py into a shared object of its own in a temporary directory; it is not linked
// into libfiducials_b200.so.  hs_calibrate_ro runs the stages in the order fid_calibrate_camera_ro enqueues them, with the same
// per-view and per-point functions; only the reduced system is solved differently: a plain dense Cholesky here, the blocked
// tensor-core kernels of calib_dense.cuh on the device.
#include "../../fiducials_b200/csrc/calib.cuh"

#include <string.h>

#include <vector>

using namespace fid;

namespace {

// Lower Cholesky of the m x m row-major matrix A in place; false on a non-positive pivot.
bool dense_cholesky(std::vector<double>& A, int m) {
    for (int j = 0; j < m; j++) {
        double s = A[(size_t)j * m + j];
        for (int k = 0; k < j; k++) s -= A[(size_t)j * m + k] * A[(size_t)j * m + k];
        if (!(s > 0.0)) return false;
        const double d = sqrt(s);
        A[(size_t)j * m + j] = d;
        for (int i = j + 1; i < m; i++) {
            double t = A[(size_t)i * m + j];
            for (int k = 0; k < j; k++) t -= A[(size_t)i * m + k] * A[(size_t)j * m + k];
            A[(size_t)i * m + j] = t / d;
        }
    }
    return true;
}
void forward(const std::vector<double>& L, int m, double* x) {
    for (int i = 0; i < m; i++) {
        double s = x[i];
        for (int k = 0; k < i; k++) s -= L[(size_t)i * m + k] * x[k];
        x[i] = s / L[(size_t)i * m + i];
    }
}
void backward(const std::vector<double>& L, int m, double* x) {
    for (int i = m - 1; i >= 0; i--) {
        double s = x[i];
        for (int k = i + 1; k < m; k++) s -= L[(size_t)k * m + i] * x[k];
        x[i] = s / L[(size_t)i * m + i];
    }
}

}  // namespace

extern "C" {

// The input is valid and released (every view holds the same n points, 1 <= fixed <= n - 2; fid_calibrate_camera_ro checks it).
// obj_in: the board [n][3]; img [nv][n][2].  Returns 0, the FID_CALIB_E_* status of a view cv2 raises on, or 8 (a non-positive
// pivot).  out: as hs_calibrate (23 doubles); rvecs, tvecs [nv][3], std_ext [nv][6], pve [nv], steps[2048], new_obj [n][3]
// (float) and std_obj [n][3].
int hs_calibrate_ro(int nv, int n, const float* obj_in, const float* img, int width, int height, const double* K, const double* D, int flags, int fixed,
                    int max_iter, double eps, double* out, double* rvecs, double* tvecs, double* std_ext, double* pve, unsigned char* steps, float* new_obj,
                    double* std_obj) {
    const int total = n * nv, m = 9 + 3 * n;
    const bool use_guess = flags & FID_CALIB_USE_INTRINSIC_GUESS_;
    std::vector<float> board(obj_in, obj_in + (size_t)n * 3);
    if (!use_guess)
        for (int i = 0; i < n; i++) board[3 * i + 2] = 0.0f;
    double aspect = 0.0;
    if (flags & FID_CALIB_FIX_ASPECT_RATIO_) aspect = K ? K[0] / K[4] : 1.0;
    double init[9] = {0, 0, (width - 1) * 0.5, (height - 1) * 0.5, 0, 0, 0, 0, 0};
    if (use_guess) {
        const double A[9] = {K[0], K[4], K[2], K[5], D[0], D[1], D[2], D[3], D[4]};
        memcpy(init, A, sizeof(init));
    } else {
        std::vector<double> ab((size_t)6 * nv);
        for (int v = 0; v < nv; v++)
            if (!calib_view_homography(n, board.data(), img + (size_t)2 * n * v, init[2], init[3], ab.data() + 6 * v)) return 3;
        double t[5];
        for (int k = 0; k < 5; k++) {
            double s = 0.0;
            for (int v = 0; v < nv; v++) {
                double tv[5];
                calib_view_normal2(ab.data() + 6 * v, tv);
                s += tv[k];
            }
            t[k] = s;
        }
        double A[4];
        calib_init_intrinsics(t, width, height, aspect, A);
        for (int a = 0; a < 4; a++) init[a] = A[a];
    }
    std::vector<double> p((size_t)6 * nv), pp((size_t)6 * nv), blk((size_t)CALIB_BLK * nv), fac((size_t)CALIB_FAC * nv), trial((size_t)3 * nv),
        mn((size_t)2 * n), pts((size_t)CALIB_PT * n), obj((size_t)3 * n), obj_prev((size_t)3 * n), S((size_t)m * m), r(m), Z((size_t)m * 6);
    for (int v = 0; v < nv; v++) {
        BoardPoseOut po;
        solve_board_pose(n, board.data(), img + (size_t)2 * n * v, mn.data(), calib_camera(init), &po);
        if (po.status != 1) return 5;
        for (int k = 0; k < 3; k++) {
            p[6 * v + k] = po.rvec[k];
            p[6 * v + 3 + k] = po.tvec[k];
        }
    }
    for (int k = 0; k < 3 * n; k++) obj[k] = obj_prev[k] = board[k];
    auto sum_views = [&](const std::vector<double>& a, size_t stride, int k) {
        double s = 0.0;
        for (int v = 0; v < nv; v++) s += a[stride * v + k];
        return s;
    };
    CalibLM* lm = new CalibLM;
    calib_lm_init(lm, init, flags, aspect, max_iter, eps);
    auto eval = [&](const double* in) {
        for (int v = 0; v < nv; v++) calib_view_eval(n, obj.data(), img + (size_t)2 * n * v, in, lm->aspect, p.data() + 6 * v, blk.data() + (size_t)CALIB_BLK * v);
        for (int i = 0; i < n; i++) calib_ro_point_sums(nv, n, i, obj.data(), img, in, lm->aspect, p.data(), pts.data() + (size_t)CALIB_PT * i);
    };
    // S and r at the J's parameters (in, pv, ob), the views' factors for `scale`; false on a non-positive pivot
    auto reduce = [&](const double U[45], const double gi[9], const double* in, const double* pv, const double* ob, double scale) {
        for (int v = 0; v < nv; v++)
            if (!calib_ro_view_factor(blk.data() + (size_t)CALIB_BLK * v, scale, fac.data() + (size_t)CALIB_FAC * v)) return false;
        for (int a = 0; a < m; a++) {
            r[a] = calib_ro_grad(a, n, fixed, lm->mask, gi, pts.data());
            for (int b = 0; b <= a; b++) S[(size_t)a * m + b] = calib_ro_entry(a, b, n, fixed, lm->mask, U, pts.data(), scale);
        }
        for (int v = 0; v < nv; v++) {
            const double* f = fac.data() + (size_t)CALIB_FAC * v;
            calib_ro_z_intrinsics(blk.data() + (size_t)CALIB_BLK * v, f, lm->mask, (double(*)[6])Z.data());
            for (int i = 0; i < n; i++)
                calib_ro_z_point(ob + 3 * i, img + 2 * ((size_t)n * v + i), in, lm->aspect, pv + 6 * v, f, i, n, fixed, (double(*)[6])(Z.data() + 6 * (9 + 3 * i)));
            for (int a = 0; a < m; a++) {
                double s = 0.0;
                for (int j = 0; j < 6; j++) s += Z[6 * a + j] * f[CALIB_FAC_H + j];
                r[a] -= s;
                for (int b = 0; b <= a; b++) {
                    double t = 0.0;
                    for (int j = 0; j < 6; j++) t += Z[6 * a + j] * Z[6 * b + j];
                    S[(size_t)a * m + b] -= t;
                }
            }
        }
        return dense_cholesky(S, m);
    };
    const int max_steps = 2 * max_iter + 20;
    int rc = 0;
    for (int s = 0; s < max_steps && lm->state != 2; s++) {
        const int state = lm->state;
        if (state == 0) {
            eval(lm->in);
            pp = p;
            obj_prev = obj;
            for (int k = 0; k < 45; k++) lm->U[k] = sum_views(blk, CALIB_BLK, CALIB_U + k);
            for (int k = 0; k < 9; k++) lm->g[k] = sum_views(blk, CALIB_BLK, CALIB_GI + k);
            lm->err = sum_views(blk, CALIB_BLK, CALIB_COST);
            calib_lm_after_eval(lm, lm->err);
            lm->state = 1;
        }
        if (!reduce(lm->U, lm->g, lm->in_prev, pp.data(), obj_prev.data(), 1.0 + calib_pow10(lm->lg))) {
            rc = 8;
            break;
        }
        forward(S, m, r.data());
        backward(S, m, r.data());
        calib_lm_trial_intrinsics(lm, r.data());
        double on[2];
        calib_ro_obj_trial(n, fixed, obj_prev.data(), r.data() + 9, obj.data(), on);
        for (int v = 0; v < nv; v++)
            calib_ro_view_trial(n, obj_prev.data(), obj.data(), r.data() + 9, img + (size_t)2 * n * v, lm->in_prev, lm->in, lm->aspect, blk.data() + (size_t)CALIB_BLK * v,
                                fac.data() + (size_t)CALIB_FAC * v, lm->dint, pp.data() + 6 * v, p.data() + 6 * v, trial.data() + 3 * v);
        calib_lm_decide(lm, sum_views(trial, 3, 0), sum_views(trial, 3, 1) + on[0], sum_views(trial, 3, 2) + on[1]);
    }
    // final parameters: undamped blocks, S^-1's diagonal, Z^T S^-1 Z per view, standard deviations and errors
    if (!rc) {
        eval(lm->in);
        double U[45], gi[9];
        for (int k = 0; k < 45; k++) U[k] = sum_views(blk, CALIB_BLK, CALIB_U + k);
        for (int k = 0; k < 9; k++) gi[k] = sum_views(blk, CALIB_BLK, CALIB_GI + k);
        const double err = sum_views(blk, CALIB_BLK, CALIB_COST);
        lm->n_evals++;
        if (!reduce(U, gi, lm->in, p.data(), obj.data(), 1.0)) rc = 8;
        if (!rc) {
            const double sigma2 = err / (double)(2 * total - calib_ro_nfree(lm->mask, nv, n));
            std::vector<double> y(m);
            for (int a = 0; a < m; a++) {
                for (int k = 0; k < m; k++) y[k] = k == a ? 1.0 : 0.0;
                forward(S, m, y.data());
                double d = 0.0;
                for (int k = 0; k < m; k++) d += y[k] * y[k];
                const double sd = calib_ro_param_free(a, n, fixed, lm->mask) ? sqrt(d * sigma2) : 0.0;
                if (a < 9) out[10 + a] = sd;
                else std_obj[a - 9] = sd;
            }
            std::vector<double> T((size_t)6 * m);
            for (int v = 0; v < nv; v++) {
                const double* f = fac.data() + (size_t)CALIB_FAC * v;
                calib_ro_z_intrinsics(blk.data() + (size_t)CALIB_BLK * v, f, lm->mask, (double(*)[6])Z.data());
                for (int i = 0; i < n; i++)
                    calib_ro_z_point(obj.data() + 3 * i, img + 2 * ((size_t)n * v + i), lm->in, lm->aspect, p.data() + 6 * v, f, i, n, fixed,
                                     (double(*)[6])(Z.data() + 6 * (9 + 3 * i)));
                for (int j = 0; j < 6; j++) {
                    for (int a = 0; a < m; a++) T[(size_t)j * m + a] = Z[6 * a + j];
                    forward(S, m, T.data() + (size_t)j * m);
                }
                double M[36];
                for (int j = 0; j < 6; j++)
                    for (int k = 0; k < 6; k++) {
                        double s = 0.0;
                        for (int a = 0; a < m; a++) s += T[(size_t)j * m + a] * T[(size_t)k * m + a];
                        M[6 * j + k] = s;
                    }
                calib_ro_view_std(f, M, sigma2, std_ext + 6 * v);
                pve[v] = sqrt(blk[(size_t)CALIB_BLK * v + CALIB_COST] / n);
                for (int k = 0; k < 3; k++) {
                    rvecs[3 * v + k] = p[6 * v + k];
                    tvecs[3 * v + k] = p[6 * v + 3 + k];
                }
            }
            out[0] = sqrt(err / total);
            for (int a = 0; a < 9; a++) out[1 + a] = lm->in[a];
            for (int k = 0; k < 3 * n; k++) new_obj[k] = (float)obj[k];
        }
    }
    out[19] = lm->iters;
    out[20] = lm->n_steps;
    out[21] = lm->n_evals;
    memcpy(steps, lm->steps, lm->n_steps < CALIB_MAX_STEPS ? lm->n_steps : CALIB_MAX_STEPS);
    delete lm;
    return rc;
}

}  // extern "C"
