// Bundle adjustment of a fiducial map from recorded marker corners (fid_map_bundle_adjust, DESIGN.md f16).
//
// NEW -- the reference folds per-marker poses into the map one message at a time (map.cpp:152-320) and never revisits an
// observation.  Parity is stated here and checked against scipy.optimize.least_squares on the same residuals.
//
//   unknowns   every used frame's camera-from-map pose (R_f, t_f) and every free map entry's map-from-marker pose (R_m, t_m)
//   gauge      entries with variance 0 stay fixed (the origin fiducial of autoInit / add_fiducial, map.cpp:483, :526)
//   residual   per observation of marker m in frame f, 8 values: pi(K, D, R_f (R_m o_k + t_m) + t_f) - c_fk, k = 0..3, pi =
//              cv::projectPoints (plumb_bob), o_k = getSingleMarkerObjectPoints(len) as fid_pose builds it (float side / 2.f)
//   update     R <- R Exp(-x_theta), t <- t - x_t for frames and markers alike, x the CvLevMarq step (calib.cuh's schedule,
//              diagonals damped by 1 + lambda); the d/d theta columns are project_point's with dR/dr = R [e_k]x
//   step       the frames are eliminated: per frame U_f, g_f and per observation W_o = J_f^T J_m; per free marker V_m, g_m;
//              S = blockdiag(V) - sum_f W_f^T U_f^-1 W_f over the free markers (dense, 6M x 6M), factored by calib_dense.cuh
//              on the device (a plain Cholesky in the host build), then the frames back-substituted
//   init       per frame solvePnP(ITERATIVE) of its mapped markers as one board (board_pnp.cuh, solve_board_pose; the object
//              points are the map-frame corners narrowed to float32 -- cv2's answer), unless one marker's own pose (fid_pose's
//              solve_marker_pose) composed with its map pose reprojects the frame's corners better.  A map as the fold leaves it is nearly but not exactly planar; there solvePnP takes its non-planar DLT,
//              which is poorly conditioned and can put the camera metres off, while a single marker's pose is always usable
//
// Every sum runs in a fixed order (observations of a frame in detection order, of a marker in frame order, frames in frame
// order), and cos, sin, acos are calib.cuh's, so the device and the host build compute the same bits up to the Cholesky of S.
#pragma once
#include <stdint.h>

#include <algorithm>
#include <unordered_map>
#include <vector>

#include "calib.cuh"

namespace fid {

#define BA_MAX_FREE 1024        // free markers: S is at most 6144 x 6144
#define BA_MAX_FRAMES 65536
#define BA_MAX_OBS (1 << 22)
#define BA_MAX_STEPS(max_iter) (2 * (max_iter) + 20)  // CvLevMarq's trial steps of a run (calib.cuh)

// Per observation (doubles): U = Jf^T Jf upper 21, W = Jf^T Jm 6x6 row-major (frame rows, marker columns), V = Jm^T Jm upper 21,
// gf = Jf^T e, gm = Jm^T e, cost = e^T e
#define BA_O_U 0
#define BA_O_W 21
#define BA_O_V 57
#define BA_O_GF 78
#define BA_O_GM 84
#define BA_O_C 90
#define BA_OBS 91
// Per frame: U upper 21, g 6, cost 1, L of the damped U packed 21, h = L^-1 g 6, trial cost, |x|^2, |p|^2
#define BA_F_U 0
#define BA_F_G 21
#define BA_F_C 27
#define BA_F_L 28
#define BA_F_H 49
#define BA_F_T 55
#define BA_FRM 58
// Per free marker: V upper 21, g 6, |x|^2, |p|^2
#define BA_M_V 0
#define BA_M_G 21
#define BA_M_T 27
#define BA_MRK 29

// getSingleMarkerObjectPoints (aruco_detect.cpp:151-161) as fid_pose builds it: TL, TR, BR, BL at +-(float)len / 2.f.
FID_HD void ba_object_points(double len, double o[4][3]) {
    const float hf = (float)len / 2.f;
    const double h = hf;
    const double c[4][3] = {{-h, h, 0}, {h, h, 0}, {h, -h, 0}, {-h, -h, 0}};
    for (int k = 0; k < 4; k++)
        for (int c3 = 0; c3 < 3; c3++) o[k][c3] = c[k][c3];
}

// dR/dtheta_k = R [e_k]x in project_point's dRdr layout (dRdr[k * 9 + i] = d R[i] / d theta_k).
FID_HD void ba_drdtheta(const double R[9], double dRdr[27]) {
    for (int k = 0; k < 3; k++)
        for (int i = 0; i < 3; i++) {
            // row i of R [e_k]x: column j of [e_k]x is e_k x e_j
            const double r0 = R[3 * i], r1 = R[3 * i + 1], r2 = R[3 * i + 2];
            double* d = dRdr + 9 * k + 3 * i;
            if (k == 0) { d[0] = 0.0; d[1] = r2; d[2] = -r1; }
            else if (k == 1) { d[0] = -r2; d[1] = 0.0; d[2] = r0; }
            else { d[0] = r1; d[1] = -r0; d[2] = 0.0; }
        }
}

// One corner: e = pi(R_f (R_m o + t_m) + t_f) - c and, when Jf is non-null, d e / d (theta_f, t_f) and d e / d (theta_m, t_m).
// pf = {unused x3, t_f}; dRf = ba_drdtheta(R_f).
FID_HD void ba_corner(const double o[3], const float c[2], const Camera& cam, const double Rf[9], const double* dRf, const double pf[6], const double Rm[9],
                      const double tm[3], double e[2], double Jf[2][6], double Jm[2][6]) {
    double X[3];
    for (int i = 0; i < 3; i++) X[i] = Rm[3 * i] * o[0] + Rm[3 * i + 1] * o[1] + Rm[3 * i + 2] * o[2] + tm[i];
    double uv[2];
    project_point(X[0], X[1], X[2], Rf, dRf, pf, cam, uv, Jf);
    e[0] = uv[0] - c[0];
    e[1] = uv[1] - c[1];
    if (!Jf) return;
    // d e / d t_m = d e / d t_f R_f; d e / d theta_m,k = d e / d t_m R_m (e_k x o)
    for (int r = 0; r < 2; r++)
        for (int j = 0; j < 3; j++) Jm[r][3 + j] = Jf[r][3] * Rf[j] + Jf[r][4] * Rf[3 + j] + Jf[r][5] * Rf[6 + j];
    const double ex[3][3] = {{0.0, -o[2], o[1]}, {o[2], 0.0, -o[0]}, {-o[1], o[0], 0.0}};
    for (int k = 0; k < 3; k++) {
        double v[3];
        for (int i = 0; i < 3; i++) v[i] = Rm[3 * i] * ex[k][0] + Rm[3 * i + 1] * ex[k][1] + Rm[3 * i + 2] * ex[k][2];
        for (int r = 0; r < 2; r++) Jm[r][k] = Jm[r][3] * v[0] + Jm[r][4] * v[1] + Jm[r][5] * v[2];
    }
}

// One observation (4 corners, in corner order): its block (layout BA_O_*) at frame pose pf = {R 9, t 3} and marker pose pm.
FID_HD void ba_obs_eval(const double o[4][3], const float* corners, const Camera& cam, const double* pf, const double* pm, double* blk) {
    double dRf[27], p6[6] = {0, 0, 0, pf[9], pf[10], pf[11]};
    ba_drdtheta(pf, dRf);
    for (int k = 0; k < BA_OBS; k++) blk[k] = 0.0;
    for (int k = 0; k < 4; k++) {
        double e[2], Jf[2][6], Jm[2][6];
        ba_corner(o[k], corners + 2 * k, cam, pf, dRf, p6, pm, pm + 9, e, Jf, Jm);
        for (int a = 0, u = 0; a < 6; a++)
            for (int b = a; b < 6; b++, u++) {
                blk[BA_O_U + u] += Jf[0][a] * Jf[0][b] + Jf[1][a] * Jf[1][b];
                blk[BA_O_V + u] += Jm[0][a] * Jm[0][b] + Jm[1][a] * Jm[1][b];
            }
        for (int a = 0; a < 6; a++)
            for (int b = 0; b < 6; b++) blk[BA_O_W + 6 * a + b] += Jf[0][a] * Jm[0][b] + Jf[1][a] * Jm[1][b];
        for (int a = 0; a < 6; a++) {
            blk[BA_O_GF + a] += Jf[0][a] * e[0] + Jf[1][a] * e[1];
            blk[BA_O_GM + a] += Jm[0][a] * e[0] + Jm[1][a] * e[1];
        }
        blk[BA_O_C] += e[0] * e[0] + e[1] * e[1];
    }
}

// One observation's e^T e (4 corners, in corner order).
FID_HD double ba_obs_cost(const double o[4][3], const float* corners, const Camera& cam, const double* pf, const double* pm) {
    const double p6[6] = {0, 0, 0, pf[9], pf[10], pf[11]};
    double s = 0.0;
    for (int k = 0; k < 4; k++) {
        double e[2];
        ba_corner(o[k], corners + 2 * k, cam, pf, nullptr, p6, pm, pm + 9, e, nullptr, nullptr);
        s += e[0] * e[0] + e[1] * e[1];
    }
    return s;
}

// Z_o = L^-1 W_o (6x6 row-major) from the frame's factor L (packed lower).
FID_HD void ba_obs_z(const double* L, const double* W, double Z[36]) {
    for (int c = 0; c < 6; c++) {
        double w[6], z[6];
        for (int a = 0; a < 6; a++) w[a] = W[6 * a + c];
        calib_ro_lsolve6(L, w, z);
        for (int a = 0; a < 6; a++) Z[6 * a + c] = z[a];
    }
}

// The trial pose q = p Exp(-x_theta), t - x_t of a pose p = {R 9, t 3}, and {|x|^2, |p|^2} with |p|^2 = angle(R)^2 + |t|^2.
FID_HD void ba_pose_step(const double* p, const double x[6], double* q, double out[2]) {
    double w[3] = {-x[0], -x[1], -x[2]}, E[9];
    rodrigues_v2m(w, E, nullptr);
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) q[3 * i + j] = p[3 * i] * E[j] + p[3 * i + 1] * E[3 + j] + p[3 * i + 2] * E[6 + j];
    double dn = 0.0, tn = 0.0;
    for (int i = 0; i < 3; i++) q[9 + i] = p[9 + i] - x[3 + i];
    for (int i = 0; i < 6; i++) dn += x[i] * x[i];
    for (int i = 0; i < 3; i++) tn += p[9 + i] * p[9 + i];
    double c = (p[0] + p[4] + p[8] - 1.0) * 0.5;
    c = c > 1.0 ? 1.0 : (c < -1.0 ? -1.0 : c);
    const double th = det_acos(c);
    out[0] = dn;
    out[1] = th * th + tn;
}

// Standard deviations of a free marker's (theta, t) from diag(S^-1) and sigma^2.
FID_HD void ba_std(const double* diag, double sigma2, double out[6]) {
    for (int k = 0; k < 6; k++) out[k] = sqrt(diag[k] * sigma2);
}

// The sum of squared reprojection errors of the n points obj (float32, map frame) / img at the camera-from-map pose {R 9, t 3};
// -1 when a point is not in front of the camera.  For coplanar points the pose mirrored through the plane with every depth
// negated reprojects exactly as well, so the depth test is what tells the two apart.
FID_HD double ba_reproj(int n, const float* obj, const float* img, const Camera& cam, const double* pose) {
    const double p6[6] = {0, 0, 0, pose[9], pose[10], pose[11]};
    double s[2];
    board_sum<2>(n, [&](int i, double v[2]) {
        double uv[2];
        const double X = obj[3 * i], Y = obj[3 * i + 1], Z = obj[3 * i + 2];
        project_point(X, Y, Z, pose, nullptr, p6, cam, uv, nullptr);
        const double a = uv[0] - img[2 * i], b = uv[1] - img[2 * i + 1];
        v[0] = a * a + b * b;
        v[1] = pose[6] * X + pose[7] * Y + pose[8] * Z + p6[5] > 0.0 ? 0.0 : 1.0;
    }, s);
    return s[1] == 0.0 ? s[0] : -1.0;
}

// A frame's initial pose (see the top of this file): n markers, obj [n][4][3] their map-frame corners (float32), img [n][4][2]
// their corners, mn [4n][2] scratch, len_f [n] their lengths as fid_pose narrows them, mpose [n][12] their map poses.  Device:
// called by the 32 lanes of a warp together (every lane computes the same bits).  False when no candidate has every corner in
// front of the camera and a finite error.  start (optional): 0 when the board pose was taken, 1 + j for marker j's own pose.
FID_HD bool ba_init_frame(int n, const float* obj, const float* img, double* mn, const Camera& cam, const float* len_f, const double* mpose, double pose[12],
                          int* start = nullptr) {
    double eb = -1.0, ec = -1.0, cand[12], bpose[12];
    int jc = -1;
    BoardPoseOut bo;
    solve_board_pose(4 * n, obj, img, mn, cam, &bo);
    if (bo.status == 1) {
        rodrigues_v2m(bo.rvec, bpose, nullptr);
        for (int k = 0; k < 3; k++) bpose[9 + k] = bo.tvec[k];
        const double e = ba_reproj(4 * n, obj, img, cam, bpose);
        if (e >= 0.0 && e < 1e300) eb = e;
    }
    for (int j = 0; j < n; j++) {  // T_cam_map = T_cam_marker T_map_marker^-1
        PoseOut po;
        solve_marker_pose(img + 8 * j, cam, len_f[j], (double)len_f[j], &po);
        double Rc[9];
        rodrigues_v2m(po.rvec, Rc, nullptr);
        const double* Rm = mpose + 12 * j;
        for (int a = 0; a < 3; a++)
            for (int b = 0; b < 3; b++) cand[3 * a + b] = Rc[3 * a] * Rm[3 * b] + Rc[3 * a + 1] * Rm[3 * b + 1] + Rc[3 * a + 2] * Rm[3 * b + 2];
        for (int a = 0; a < 3; a++)
            cand[9 + a] = po.tvec[a] - (cand[3 * a] * Rm[9] + cand[3 * a + 1] * Rm[10] + cand[3 * a + 2] * Rm[11]);
        const double e = ba_reproj(4 * n, obj, img, cam, cand);
        if (e >= 0.0 && e < 1e300 && (ec < 0.0 || e < ec)) {
            ec = e;
            jc = j;
            for (int k = 0; k < 12; k++) pose[k] = cand[k];
        }
    }
    // the board pose (cv2's) unless a marker's pose reprojects the frame's corners better
    const bool board = eb >= 0.0 && !(ec >= 0.0 && ec < eb);
    if (board)
        for (int k = 0; k < 12; k++) pose[k] = bpose[k];
    if (start) *start = board ? 0 : 1 + jc;
    return eb >= 0.0 || ec >= 0.0;
}

// CvLevMarq state of a bundle adjustment (calib.cuh's schedule).
struct BaLM {
    int state;  // 0 evaluate J, 1 trial step from the last J, 2 done
    int lg, iters, max_iter, n_steps, n_evals;
    int converged;  // the run ended on the relative-step test (not on max_iter)
    double eps, err, prev_err, err0;
};

FID_HD void ba_lm_init(BaLM* s, int max_iter, double eps) {
    s->state = 0;
    s->lg = -3;
    s->iters = s->n_steps = s->n_evals = s->converged = 0;
    s->max_iter = max_iter;
    s->eps = eps;
    s->err = s->prev_err = s->err0 = 0.0;
}

FID_HD void ba_lm_after_eval(BaLM* s, double err) {
    if (s->n_evals == 0) s->err0 = err;
    s->n_evals++;
    s->err = s->prev_err = err;
    s->state = 1;
}

FID_HD void ba_lm_decide(BaLM* s, double err, double dn, double pn) {
    s->err = err;
    lm_schedule_decide(&s->state, &s->lg, &s->iters, s->max_iter, s->eps, err, s->prev_err, dn, pn);
    s->n_steps++;
    if (s->state == 2) s->converged = sqrt(dn) / (sqrt(pn) + 2.220446049250313e-16) < s->eps;
}

// The map-frame corners R_m o_k + t_m of a marker, narrowed to float32 (the object points of the frame's board).
FID_HD void ba_map_corners(const double R[9], const double t[3], const double o[4][3], float out[12]) {
    for (int k = 0; k < 4; k++)
        for (int i = 0; i < 3; i++) out[3 * k + i] = (float)(R[3 * i] * o[k][0] + R[3 * i + 1] * o[k][1] + R[3 * i + 2] * o[k][2] + t[i]);
}

// ---- host: which observations count (shared by fid_map_bundle_adjust and the host build) -----------------------------------
// Frame statuses (fid_map_bundle_adjust's frame_status)
#define BA_FRAME_NONE 0       // no mapped marker
#define BA_FRAME_USED 1
#define BA_FRAME_UNREACHED 2  // not connected to a fixed entry through co-visibility
#define BA_FRAME_INIT 3       // no initial pose (no candidate with a finite reprojection error)

struct BaPlan {
    // stage 1 (ba_plan_observations): candidate frames and their mapped observations in detection order
    int n_dropped_unmapped = 0, n_dropped_duplicate = 0;
    std::vector<int32_t> status;            // per input frame
    std::vector<int32_t> cand;              // candidate frames (input index), in order
    std::vector<int32_t> c_off;             // CSR per candidate frame into c_slot / c_src
    std::vector<int32_t> c_slot, c_src;     // map slot, index j + f * max_markers of the detection
    // stage 2 (ba_plan_solve): after the initial poses
    int n_free = 0, n_unreached_markers = 0, n_unreached_frames = 0, n_init_failed = 0;
    std::vector<int32_t> slot_free;         // per map slot: free index or -1
    std::vector<int32_t> free_slot;         // free index -> slot
    std::vector<int32_t> frames;            // used frame -> candidate index
    std::vector<int32_t> f_off;             // CSR per used frame into the observations
    std::vector<int32_t> o_slot, o_src, o_free, o_frame;  // per observation
    std::vector<int32_t> m_off, m_obs;      // CSR per free marker: its observations in frame order
    std::vector<int32_t> b_ab, b_off, b_pair;  // nonzero blocks (a <= b as a | b << 16), per block the (obs of a, obs of b) pairs in frame order
};

// Stage 1.  ids of the map slots; a detection counts when its id is in the map and appears once in its frame.
inline void ba_plan_observations(int n_frames, const int32_t* counts, const int32_t* ids, int max_markers, int n_slots, const int32_t* slot_ids, BaPlan* P) {
    std::unordered_map<int32_t, int32_t> slot;
    for (int s = 0; s < n_slots; s++) slot[slot_ids[s]] = s;
    P->status.assign(n_frames, BA_FRAME_NONE);
    P->c_off.assign(1, 0);
    std::unordered_map<int32_t, int> seen;
    for (int f = 0; f < n_frames; f++) {
        const int32_t* fid = ids + (size_t)f * max_markers;
        seen.clear();
        for (int j = 0; j < counts[f]; j++) seen[fid[j]]++;
        const size_t before = P->c_slot.size();
        for (int j = 0; j < counts[f]; j++) {
            auto it = slot.find(fid[j]);
            if (it == slot.end()) {
                P->n_dropped_unmapped++;
                continue;
            }
            if (seen[fid[j]] > 1) {
                P->n_dropped_duplicate++;
                continue;
            }
            P->c_slot.push_back(it->second);
            P->c_src.push_back((int32_t)((size_t)f * max_markers + j));
        }
        if (P->c_slot.size() > before) {
            P->cand.push_back(f);
            P->c_off.push_back((int32_t)P->c_slot.size());
        }
    }
}

// Stage 2.  init_ok[c] = the initial pose of candidate frame c succeeded; fixed[s] = slot s has variance 0.
inline void ba_plan_solve(int n_slots, const uint8_t* fixed, const uint8_t* init_ok, BaPlan* P) {
    const int nc = (int)P->cand.size();
    std::vector<int> parent(n_slots);
    for (int s = 0; s < n_slots; s++) parent[s] = s;
    auto find = [&](int x) {
        while (parent[x] != x) x = parent[x] = parent[parent[x]];
        return x;
    };
    for (int c = 0; c < nc; c++) {
        if (!init_ok[c]) continue;
        for (int k = P->c_off[c] + 1; k < P->c_off[c + 1]; k++) {
            const int a = find(P->c_slot[P->c_off[c]]), b = find(P->c_slot[k]);
            if (a != b) parent[a] = b;
        }
    }
    std::vector<uint8_t> root_fixed(n_slots, 0);
    for (int s = 0; s < n_slots; s++)
        if (fixed[s]) root_fixed[find(s)] = 1;
    std::vector<uint8_t> observed(n_slots, 0);
    P->frames.clear();
    P->f_off.assign(1, 0);
    for (int c = 0; c < nc; c++) {
        const int f = P->cand[c];
        if (!init_ok[c]) {
            P->status[f] = BA_FRAME_INIT;
            P->n_init_failed++;
            continue;
        }
        if (!root_fixed[find(P->c_slot[P->c_off[c]])]) {
            P->status[f] = BA_FRAME_UNREACHED;
            P->n_unreached_frames++;
            continue;
        }
        P->status[f] = BA_FRAME_USED;
        P->frames.push_back(c);
        for (int k = P->c_off[c]; k < P->c_off[c + 1]; k++) {
            P->o_slot.push_back(P->c_slot[k]);
            P->o_src.push_back(P->c_src[k]);
            P->o_frame.push_back((int32_t)P->frames.size() - 1);
            observed[P->c_slot[k]] = 1;
        }
        P->f_off.push_back((int32_t)P->o_slot.size());
    }
    P->slot_free.assign(n_slots, -1);
    P->free_slot.clear();
    P->n_unreached_markers = 0;
    for (int s = 0; s < n_slots; s++) {
        if (fixed[s]) continue;
        if (!observed[s]) {
            P->n_unreached_markers++;
            continue;
        }
        P->slot_free[s] = (int32_t)P->free_slot.size();
        P->free_slot.push_back(s);
    }
    P->n_free = (int)P->free_slot.size();
    const size_t no = P->o_slot.size();
    P->o_free.resize(no);
    P->m_off.assign((size_t)P->n_free + 1, 0);
    for (size_t o = 0; o < no; o++) {
        P->o_free[o] = P->slot_free[P->o_slot[o]];
        if (P->o_free[o] >= 0) P->m_off[P->o_free[o] + 1]++;
    }
    for (int m = 0; m < P->n_free; m++) P->m_off[m + 1] += P->m_off[m];
    P->m_obs.assign(P->m_off.back(), 0);
    {
        std::vector<int32_t> fill(P->m_off.begin(), P->m_off.end() - 1);
        for (size_t o = 0; o < no; o++)
            if (P->o_free[o] >= 0) P->m_obs[fill[P->o_free[o]]++] = (int32_t)o;
    }
    // nonzero blocks of S: (a, a) for every free marker, (a, b) for every pair seen together; pairs in frame order
    std::unordered_map<uint32_t, std::vector<int32_t>> blocks;
    for (int m = 0; m < P->n_free; m++) {
        auto& v = blocks[(uint32_t)m | ((uint32_t)m << 16)];
        for (int k = P->m_off[m]; k < P->m_off[m + 1]; k++) {
            v.push_back(P->m_obs[k]);
            v.push_back(P->m_obs[k]);
        }
    }
    const int nf = (int)P->frames.size();
    for (int f = 0; f < nf; f++)
        for (int i = P->f_off[f]; i < P->f_off[f + 1]; i++)
            for (int j = P->f_off[f]; j < P->f_off[f + 1]; j++) {
                const int a = P->o_free[i], b = P->o_free[j];
                if (a < 0 || b < 0 || a >= b) continue;
                auto& v = blocks[(uint32_t)a | ((uint32_t)b << 16)];
                v.push_back(i);
                v.push_back(j);
            }
    P->b_ab.clear();
    for (auto& kv : blocks) P->b_ab.push_back((int32_t)kv.first);
    std::sort(P->b_ab.begin(), P->b_ab.end());
    P->b_off.assign(1, 0);
    P->b_pair.clear();
    for (int32_t k : P->b_ab) {
        const auto& v = blocks[(uint32_t)k];
        P->b_pair.insert(P->b_pair.end(), v.begin(), v.end());
        P->b_off.push_back((int32_t)(P->b_pair.size() / 2));
    }
}

// The marker length of an id: its override, else fiducial_len.
FID_HD double ba_marker_len(int32_t id, double fiducial_len, int n_override, const int32_t* override_ids, const double* override_lens) {
    for (int k = 0; k < n_override; k++)
        if (override_ids[k] == id) return override_lens[k];
    return fiducial_len;
}

}  // namespace fid
