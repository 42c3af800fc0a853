// CPU harness for fiducials_b200/csrc/map_ba.cuh (fid_map_bundle_adjust).  TEST INFRASTRUCTURE ONLY.  Compiled with g++ by
// tests/map_ba_cases.py into a shared object of its own in a temporary directory; it is not linked into libfiducials_b200.so.
// hs_map_ba runs the stages in the order fid_map_bundle_adjust enqueues them, with the same per-observation, per-frame and
// per-block functions and the same summation orders; only the reduced system is factored differently: a plain dense Cholesky
// here, the blocked tensor-core kernels of calib_dense.cuh on the device.
#include "../../fiducials_b200/csrc/map_ba.cuh"

#include <string.h>

#include <vector>

using namespace fid;

namespace {

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

// One corner's residual and Jacobians (for the derivative tests).  pf, pm = {R 9, t 3}; out: e 2, Jf 12, Jm 12.
void hs_ba_corner(const double* o, const float* c, const double* K, const double* D, const double* pf, const double* pm, double* out) {
    const Camera cam{K[0], K[4], K[2], K[5], D[0], D[1], D[2], D[3], D[4]};
    double dRf[27], p6[6] = {0, 0, 0, pf[9], pf[10], pf[11]}, e[2], Jf[2][6], Jm[2][6];
    ba_drdtheta(pf, dRf);
    ba_corner(o, c, cam, pf, dRf, p6, pm, pm + 9, e, Jf, Jm);
    out[0] = e[0];
    out[1] = e[1];
    for (int r = 0; r < 2; r++)
        for (int j = 0; j < 6; j++) {
            out[2 + 6 * r + j] = Jf[r][j];
            out[14 + 6 * r + j] = Jm[r][j];
        }
}

// The whole solve.  Map slots: slot_ids [n_slots], fixed [n_slots] (variance 0), poses [n_slots][12] (R row-major, t; updated in
// place for the free entries).  Frames: counts [n_frames], ids [n_frames][max_markers], corners [n_frames][max_markers][8].
// Outputs: rvecs, tvecs [n_frames][3] (0 for unused frames), status [n_frames], std [n_slots][6] (0 for fixed and unreached),
// stats [16]: initial rms, final rms, iterations, steps, frames used, free markers, observations, unmapped, duplicate, unreached
// frames, unreached markers, init failures, converged (the relative-step test ended the run).  max_iter <= 0: only the initial poses (rvecs, tvecs of every frame with a mapped
// marker).  Returns 0, or 1 on a non-positive pivot, 2 without a fixed entry.
int hs_map_ba(int n_slots, const int32_t* slot_ids, const uint8_t* fixed, double* poses, int n_frames, const int32_t* counts, const int32_t* ids,
              const float* corners, int max_markers, const double* K, const double* D, double fiducial_len, int n_override, const int32_t* override_ids,
              const double* override_lens, int max_iter, double eps, double* rvecs, double* tvecs, int32_t* status, double* std_out, double* stats) {
    const Camera cam{K[0], K[4], K[2], K[5], D[0], D[1], D[2], D[3], D[4]};
    memset(stats, 0, sizeof(double) * 16);
    for (int f = 0; f < n_frames; f++)
        for (int k = 0; k < 3; k++) rvecs[3 * f + k] = tvecs[3 * f + k] = 0.0;
    memset(std_out, 0, sizeof(double) * 6 * n_slots);
    bool any_fixed = false;
    for (int s = 0; s < n_slots; s++) any_fixed |= fixed[s] != 0;
    if (!any_fixed) return 2;
    BaPlan P;
    ba_plan_observations(n_frames, counts, ids, max_markers, n_slots, slot_ids, &P);
    std::vector<double> slot_obj((size_t)n_slots * 12);
    for (int s = 0; s < n_slots; s++) {
        double o[4][3];
        ba_object_points(ba_marker_len(slot_ids[s], fiducial_len, n_override, override_ids, override_lens), o);
        for (int k = 0; k < 4; k++)
            for (int c = 0; c < 3; c++) slot_obj[12 * s + 3 * k + c] = o[k][c];
    }
    // initial frame poses: one board per candidate frame
    const int nc = (int)P.cand.size();
    std::vector<uint8_t> init_ok(nc);
    std::vector<double> cand_pose((size_t)nc * 12);
    for (int c = 0; c < nc; c++) {
        const int n = P.c_off[c + 1] - P.c_off[c];
        std::vector<float> obj((size_t)12 * n), img((size_t)8 * n), len_f(n);
        std::vector<double> mn((size_t)8 * n), mpose((size_t)12 * n);
        for (int k = 0; k < n; k++) {
            const int o = P.c_off[c] + k, s = P.c_slot[o];
            ba_map_corners(poses + 12 * s, poses + 12 * s + 9, (const double(*)[3])(slot_obj.data() + 12 * s), obj.data() + 12 * k);
            for (int q = 0; q < 8; q++) img[8 * k + q] = corners[(size_t)8 * P.c_src[o] + q];
            for (int q = 0; q < 12; q++) mpose[12 * k + q] = poses[12 * s + q];
            len_f[k] = (float)ba_marker_len(slot_ids[s], fiducial_len, n_override, override_ids, override_lens);
        }
        init_ok[c] = ba_init_frame(n, obj.data(), img.data(), mn.data(), cam, len_f.data(), mpose.data(), cand_pose.data() + 12 * c);
    }
    std::vector<uint8_t> fx(fixed, fixed + n_slots);
    ba_plan_solve(n_slots, fx.data(), init_ok.data(), &P);
    for (int f = 0; f < n_frames; f++) status[f] = P.status[f];
    if (max_iter <= 0) {  // the initial poses of every frame with a mapped marker only
        for (int c = 0; c < nc; c++) {
            const int fi = P.cand[c];
            rodrigues_m2v(cand_pose.data() + 12 * c, rvecs + 3 * fi);
            for (int k = 0; k < 3; k++) tvecs[3 * fi + k] = cand_pose[12 * c + 9 + k];
        }
        return 0;
    }
    const int F = (int)P.frames.size(), M = P.n_free, NO = (int)P.o_slot.size();
    stats[4] = F;
    stats[5] = M;
    stats[6] = NO;
    stats[7] = P.n_dropped_unmapped;
    stats[8] = P.n_dropped_duplicate;
    stats[9] = P.n_unreached_frames;
    stats[10] = P.n_unreached_markers;
    stats[11] = P.n_init_failed;
    if (F == 0) return 0;
    std::vector<double> fp((size_t)12 * F), fp_prev((size_t)12 * F), mp((size_t)12 * M), mp_prev((size_t)12 * M);
    for (int f = 0; f < F; f++)
        for (int k = 0; k < 12; k++) fp[12 * f + k] = cand_pose[12 * P.frames[f] + k];
    for (int m = 0; m < M; m++)
        for (int k = 0; k < 12; k++) mp[12 * m + k] = poses[12 * P.free_slot[m] + k];
    // the pose of an observation's marker: a free marker's current one, else the map's
    auto mpose = [&](const std::vector<double>& cur, int o) { return P.o_free[o] >= 0 ? cur.data() + 12 * P.o_free[o] : poses + 12 * P.o_slot[o]; };
    auto obj = [&](int o) { return (const double(*)[3])(slot_obj.data() + 12 * P.o_slot[o]); };
    auto crn = [&](int o) { return corners + (size_t)8 * P.o_src[o]; };
    const int n6 = 6 * M;
    std::vector<double> blk((size_t)BA_OBS * NO), frm((size_t)BA_FRM * F), mrk((size_t)BA_MRK * M), Z((size_t)36 * NO), S((size_t)n6 * n6), r(n6);
    auto eval = [&]() {
        for (int o = 0; o < NO; o++) ba_obs_eval(obj(o), crn(o), cam, fp.data() + 12 * P.o_frame[o], mpose(mp, o), blk.data() + (size_t)BA_OBS * o);
        for (int f = 0; f < F; f++) {
            double* q = frm.data() + (size_t)BA_FRM * f;
            for (int k = 0; k < 28; k++) q[k] = 0.0;
            for (int o = P.f_off[f]; o < P.f_off[f + 1]; o++) {
                const double* b = blk.data() + (size_t)BA_OBS * o;
                for (int k = 0; k < 21; k++) q[BA_F_U + k] += b[BA_O_U + k];
                for (int k = 0; k < 6; k++) q[BA_F_G + k] += b[BA_O_GF + k];
                q[BA_F_C] += b[BA_O_C];
            }
        }
        for (int m = 0; m < M; m++) {
            double* q = mrk.data() + (size_t)BA_MRK * m;
            for (int k = 0; k < 27; k++) q[k] = 0.0;
            for (int i = P.m_off[m]; i < P.m_off[m + 1]; i++) {
                const double* b = blk.data() + (size_t)BA_OBS * P.m_obs[i];
                for (int k = 0; k < 21; k++) q[BA_M_V + k] += b[BA_O_V + k];
                for (int k = 0; k < 6; k++) q[BA_M_G + k] += b[BA_O_GM + k];
            }
        }
        double err = 0.0;
        for (int f = 0; f < F; f++) err += frm[(size_t)BA_FRM * f + BA_F_C];
        return err;
    };
    // S (lower) and r for the damping `scale`; false on a non-positive pivot of a frame's U or of S
    auto reduce = [&](double scale) {
        for (int f = 0; f < F; f++) {
            double* q = frm.data() + (size_t)BA_FRM * f;
            if (!calib_chol6(q + BA_F_U, scale, q + BA_F_L)) return false;
            calib_ro_lsolve6(q + BA_F_L, q + BA_F_G, q + BA_F_H);
        }
        for (int o = 0; o < NO; o++)
            if (P.o_free[o] >= 0) ba_obs_z(frm.data() + (size_t)BA_FRM * P.o_frame[o] + BA_F_L, blk.data() + (size_t)BA_OBS * o + BA_O_W, Z.data() + 36 * (size_t)o);
        std::fill(S.begin(), S.end(), 0.0);
        for (size_t k = 0; k < P.b_ab.size(); k++) {
            const int a = P.b_ab[k] & 0xffff, b = (P.b_ab[k] >> 16) & 0xffff;
            for (int e = 0; e < 36; e++) {
                const int i = e / 6, j = e % 6;
                double s = 0.0;
                if (a == b) {
                    const int lo = i < j ? i : j, hi = i < j ? j : i;
                    s = mrk[(size_t)BA_MRK * a + BA_M_V + lo * 6 - lo * (lo - 1) / 2 + hi - lo];
                    if (i == j) s *= scale;
                }
                for (int t = P.b_off[k]; t < P.b_off[k + 1]; t++) {
                    const double *za = Z.data() + 36 * (size_t)P.b_pair[2 * t], *zb = Z.data() + 36 * (size_t)P.b_pair[2 * t + 1];
                    double d = 0.0;
                    for (int l = 0; l < 6; l++) d += zb[6 * l + i] * za[6 * l + j];
                    s -= d;
                }
                S[(size_t)(6 * b + i) * n6 + 6 * a + j] = s;
            }
        }
        for (int m = 0; m < M; m++)
            for (int i = 0; i < 6; i++) {
                double s = mrk[(size_t)BA_MRK * m + BA_M_G + i];
                for (int t = P.m_off[m]; t < P.m_off[m + 1]; t++) {
                    const int o = P.m_obs[t];
                    const double *z = Z.data() + 36 * (size_t)o, *h = frm.data() + (size_t)BA_FRM * P.o_frame[o] + BA_F_H;
                    double d = 0.0;
                    for (int l = 0; l < 6; l++) d += z[6 * l + i] * h[l];
                    s -= d;
                }
                r[6 * m + i] = s;
            }
        return dense_cholesky(S, n6);
    };
    BaLM lm;
    ba_lm_init(&lm, max_iter, eps);
    const int max_steps = BA_MAX_STEPS(max_iter);
    int rc = 0;
    for (int s = 0; s < max_steps && lm.state != 2; s++) {
        if (lm.state == 0) {
            const double err = eval();
            fp_prev = fp;
            mp_prev = mp;
            ba_lm_after_eval(&lm, err);
        }
        if (!reduce(1.0 + calib_pow10(lm.lg))) {
            rc = 1;
            break;
        }
        forward(S, n6, r.data());
        backward(S, n6, r.data());
        // back-substitution: x_f = L^-T (h - sum_o Z_o x_m(o)), the trial poses and their norms
        double dn = 0.0, pn = 0.0, err = 0.0;
        for (int f = 0; f < F; f++) {
            double* q = frm.data() + (size_t)BA_FRM * f;
            double y[6], x[6];
            for (int k = 0; k < 6; k++) y[k] = q[BA_F_H + k];
            for (int o = P.f_off[f]; o < P.f_off[f + 1]; o++) {
                if (P.o_free[o] < 0) continue;
                const double *z = Z.data() + 36 * (size_t)o, *xm = r.data() + 6 * P.o_free[o];
                for (int k = 0; k < 6; k++) {
                    double d = 0.0;
                    for (int l = 0; l < 6; l++) d += z[6 * k + l] * xm[l];
                    y[k] -= d;
                }
            }
            calib_ro_ltsolve6(q + BA_F_L, y, x);
            ba_pose_step(fp_prev.data() + 12 * f, x, fp.data() + 12 * f, q + BA_F_T + 1);
        }
        for (int m = 0; m < M; m++) ba_pose_step(mp_prev.data() + 12 * m, r.data() + 6 * m, mp.data() + 12 * m, mrk.data() + (size_t)BA_MRK * m + BA_M_T);
        for (int f = 0; f < F; f++) {
            double c = 0.0;
            for (int o = P.f_off[f]; o < P.f_off[f + 1]; o++) c += ba_obs_cost(obj(o), crn(o), cam, fp.data() + 12 * f, mpose(mp, o));
            frm[(size_t)BA_FRM * f + BA_F_T] = c;
        }
        for (int f = 0; f < F; f++) {
            err += frm[(size_t)BA_FRM * f + BA_F_T];
            dn += frm[(size_t)BA_FRM * f + BA_F_T + 1];
            pn += frm[(size_t)BA_FRM * f + BA_F_T + 2];
        }
        for (int m = 0; m < M; m++) {
            dn += mrk[(size_t)BA_MRK * m + BA_M_T];
            pn += mrk[(size_t)BA_MRK * m + BA_M_T + 1];
        }
        ba_lm_decide(&lm, err, dn, pn);
        if (lm.state == 1) {  // rejected: the next trial starts from the J's poses again
            fp = fp_prev;
            mp = mp_prev;
        }
    }
    stats[0] = sqrt(lm.err0 / (4.0 * NO));
    stats[2] = lm.iters;
    stats[3] = lm.n_steps;
    stats[12] = lm.converged;
    if (rc) return rc;
    // final pass: undamped system at the optimum, diag(S^-1) through L^-1 e_a
    const double err = eval();
    stats[1] = sqrt(err / (4.0 * NO));
    if (!reduce(1.0)) return 1;
    const double sigma2 = err / (double)(8LL * NO - 6LL * (F + M));
    std::vector<double> y(n6);
    for (int a = 0; a < n6; a++) {
        for (int k = 0; k < n6; k++) y[k] = k == a ? 1.0 : 0.0;
        forward(S, n6, y.data());
        double d = 0.0;
        for (int k = 0; k < n6; k++) d += y[k] * y[k];
        std_out[6 * P.free_slot[a / 6] + a % 6] = sqrt(d * sigma2);
    }
    for (int m = 0; m < M; m++)
        for (int k = 0; k < 12; k++) poses[12 * P.free_slot[m] + k] = mp[12 * m + k];
    for (int f = 0; f < F; f++) {
        const int fi = P.cand[P.frames[f]];
        rodrigues_m2v(fp.data() + 12 * f, rvecs + 3 * fi);
        for (int k = 0; k < 3; k++) tvecs[3 * fi + k] = fp[12 * f + 9 + k];
    }
    return 0;
}

}  // extern "C"
