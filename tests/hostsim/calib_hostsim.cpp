// CPU harness for fiducials_b200/csrc/calib.cuh (cv::calibrateCameraExtended).  TEST INFRASTRUCTURE ONLY.
// Compiled with g++ by tests/test_hostsim_calib.py into a shared object of its own in a temporary directory, from the same header
// the kernels of fid_calib.cu are built from; it is not linked into libfiducials_b200.so.  hs_calibrate runs the stages in the
// order fid_calibrate_camera enqueues them, every sum over views in view order, so that host and device compute the same bits.
#include "../../fiducials_b200/csrc/calib.cuh"

#include <string.h>

#include <vector>

using namespace fid;

extern "C" {

// The input is valid (fid_calibrate_camera checks it).  guess: K[9] and D[5], used as fid_calibrate_camera uses them (may be
// NULL).  Returns 0 or the FID_CALIB_E_* status of a view cv2 raises on.  out: rms, fx fy cx cy k1 k2 p1 p2 k3, std[9],
// iterations, n_steps, n_evals (23 doubles); rvecs, tvecs [nv][3], std_ext [nv][6], pve [nv]; steps[2048].
int hs_calibrate(int nv, const int32_t* off, const float* obj_in, const float* img, int width, int height, const double* K, const double* D, int flags, int max_iter,
                 double eps, double* out, double* rvecs, double* tvecs, double* std_ext, double* pve, unsigned char* steps) {
    const int total = off[nv];
    const bool use_guess = flags & FID_CALIB_USE_INTRINSIC_GUESS_;
    std::vector<float> obj(obj_in, obj_in + (size_t)total * 3);
    if (!use_guess)
        for (int i = 0; i < total; i++) obj[3 * i + 2] = 0.0f;
    double aspect = 0.0;
    if (flags & FID_CALIB_FIX_ASPECT_RATIO_) aspect = K ? K[0] / K[4] : 1.0;
    double init[9] = {0, 0, (width - 1) * 0.5, (height - 1) * 0.5, 0, 0, 0, 0, 0};
    if (use_guess) {
        const double A[9] = {K[0], K[4], K[2], K[5], D[0], D[1], D[2], D[3], D[4]};
        memcpy(init, A, sizeof(init));
    } else {
        std::vector<double> ab((size_t)6 * nv);
        for (int v = 0; v < nv; v++)
            if (!calib_view_homography(off[v + 1] - off[v], obj.data() + 3 * off[v], img + 2 * off[v], init[2], init[3], ab.data() + 6 * v)) return 3;
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
    std::vector<double> p((size_t)6 * nv), pp((size_t)6 * nv), blk((size_t)CALIB_BLK * nv), sch((size_t)CALIB_SCH * nv), trial((size_t)3 * nv),
        mn((size_t)2 * total);
    for (int v = 0; v < nv; v++) {
        BoardPoseOut po;
        solve_board_pose(off[v + 1] - off[v], obj.data() + 3 * off[v], img + 2 * off[v], mn.data() + 2 * off[v], calib_camera(init), &po);
        if (po.status != 1) return 5;
        for (int k = 0; k < 3; k++) {
            p[6 * v + k] = po.rvec[k];
            p[6 * v + 3 + k] = po.tvec[k];
        }
    }
    auto sum_views = [&](const std::vector<double>& a, size_t stride, int k) {
        double s = 0.0;
        for (int v = 0; v < nv; v++) s += a[stride * v + k];
        return s;
    };
    auto eval = [&](bool final_pass, const CalibLM& lm) {
        for (int v = 0; v < nv; v++) {
            calib_view_eval(off[v + 1] - off[v], obj.data() + 3 * off[v], img + 2 * off[v], lm.in, lm.aspect, p.data() + 6 * v, blk.data() + (size_t)CALIB_BLK * v);
            if (!final_pass)
                for (int k = 0; k < 6; k++) pp[6 * v + k] = p[6 * v + k];
        }
    };
    CalibLM* lm = new CalibLM;
    calib_lm_init(lm, init, flags, aspect, max_iter, eps);
    const int max_steps = 2 * max_iter + 20;
    for (int s = 0; s < max_steps && lm->state != 2; s++) {
        const int state = lm->state;
        if (state == 0) eval(false, *lm);
        const double scale = 1.0 + calib_pow10(lm->lg);
        for (int v = 0; v < nv; v++) calib_view_schur(blk.data() + (size_t)CALIB_BLK * v, scale, sch.data() + (size_t)CALIB_SCH * v);
        if (state == 0) {
            for (int k = 0; k < 45; k++) lm->U[k] = sum_views(blk, CALIB_BLK, CALIB_U + k);
            for (int k = 0; k < 9; k++) lm->g[k] = sum_views(blk, CALIB_BLK, CALIB_GI + k);
            lm->err = sum_views(blk, CALIB_BLK, CALIB_COST);
        }
        double Q[45], q[9];
        for (int k = 0; k < 45; k++) Q[k] = sum_views(sch, CALIB_SCH, CALIB_Q + k);
        for (int k = 0; k < 9; k++) q[k] = sum_views(sch, CALIB_SCH, CALIB_QV + k);
        if (state == 0) {
            calib_lm_after_eval(lm, lm->err);
            lm->state = 1;
        }
        double dint[9];
        calib_solve_intrinsics(lm->U, lm->g, Q, q, 1.0 + calib_pow10(lm->lg), lm->mask, dint);
        calib_lm_trial_intrinsics(lm, dint);
        for (int v = 0; v < nv; v++) {
            double pv[6];
            calib_view_trial(off[v + 1] - off[v], obj.data() + 3 * off[v], img + 2 * off[v], lm->in, lm->aspect, blk.data() + (size_t)CALIB_BLK * v,
                             sch.data() + (size_t)CALIB_SCH * v, lm->dint, pp.data() + 6 * v, pv, trial.data() + 3 * v);
            for (int k = 0; k < 6; k++) p[6 * v + k] = pv[k];
        }
        calib_lm_decide(lm, sum_views(trial, 3, 0), sum_views(trial, 3, 1), sum_views(trial, 3, 2));
    }
    // final parameters: undamped blocks, S^-1, standard deviations and errors
    eval(true, *lm);
    for (int v = 0; v < nv; v++) calib_view_schur(blk.data() + (size_t)CALIB_BLK * v, 1.0, sch.data() + (size_t)CALIB_SCH * v);
    double U[45], Q[45];
    for (int k = 0; k < 45; k++) {
        U[k] = sum_views(blk, CALIB_BLK, CALIB_U + k);
        Q[k] = sum_views(sch, CALIB_SCH, CALIB_Q + k);
    }
    const double err = sum_views(blk, CALIB_BLK, CALIB_COST);
    lm->n_evals++;
    double Sinv[9][9];
    calib_schur_inverse(U, Q, lm->mask, Sinv);
    int nfree = 6 * nv;
    for (int a = 0; a < 9; a++) nfree += lm->mask[a];
    const double sigma2 = err / (double)(2 * total - nfree);
    out[0] = sqrt(err / total);
    for (int a = 0; a < 9; a++) {
        out[1 + a] = lm->in[a];
        out[10 + a] = lm->mask[a] ? sqrt(Sinv[a][a] * sigma2) : 0.0;
    }
    out[19] = lm->iters;
    out[20] = lm->n_steps;
    out[21] = lm->n_evals;
    for (int v = 0; v < nv; v++) {
        for (int k = 0; k < 3; k++) {
            rvecs[3 * v + k] = p[6 * v + k];
            tvecs[3 * v + k] = p[6 * v + 3 + k];
        }
        calib_view_std(blk.data() + (size_t)CALIB_BLK * v, sch.data() + (size_t)CALIB_SCH * v, Sinv, sigma2, std_ext + 6 * v);
        pve[v] = sqrt(blk[(size_t)CALIB_BLK * v + CALIB_COST] / (off[v + 1] - off[v]));
    }
    memcpy(steps, lm->steps, lm->n_steps < CALIB_MAX_STEPS ? lm->n_steps : CALIB_MAX_STEPS);
    delete lm;
    return 0;
}

}  // extern "C"
