// Localization against the fiducial map: one camera pose per frame from every visible mapped marker's corners (fid_map_localize,
// DESIGN.md f17).
//
// NEW -- the reference's updatePose (map.cpp:247-391) makes one camera pose per marker from that marker's 4 corners and averages
// them with heuristic variances; map.cpp:127-129 reads a `multi_error_theshold` for a multi-fiducial pose that it never computes.
// Each step below is stated so that it can be checked against cv2:
//   match     a detection counts when its id is in the map, appears once in the frame (fid_map_bundle_adjust's rule) and, with
//             max_entry_variance >= 0, the entry's variance is <= that bound; detection order is kept
//   board     per counted marker ba_object_points(len) through its entry's pose, narrowed to float32 (ba_map_corners): the
//             cv2.aruco.Board of tests/map_ba_cases.board_init_cv2
//   start     ba_init_frame: the board solvePnP, unless one marker's own pose composed with its map pose reprojects every corner
//             better; candidates with a corner behind the camera never count (a fold's map is nearly planar, and there the
//             non-planar DLT and the mirrored solution are the hazards)
//   LM        board_pose_lm from that start: what cv2.solvePnP(..., useExtrinsicGuess=True, SOLVEPNP_ITERATIVE) runs
//   cov       sigma^2 (J^T J)^-1 of the output pose (T_mapBase, or T_mapCam without a mount) under (Exp([dtheta]x) R, t + dt), J
//             analytic at the final pose: with v = X_map - t, d X_cam / d dt = -R_cm and d X_cam / d dtheta = R_cm [v]x
// Device: called by the 32 lanes of a warp together, every lane computing the same bits (board_sum's lane model).
#pragma once
#include <string.h>

#include "../../include/fiducials_b200.h"
#include "map_ba.cuh"
#include "slam.cuh"

namespace fid {

// The map slot of detection j of a frame with n detections when it counts (the match rule above), else -1.
FID_HD int loc_slot(const MapState& st, const MapEntry* e, const MapHash* h, int n, const int32_t* ids, int j, double max_entry_variance) {
    const int32_t id = ids[j];
    const int s = map_find(st, e, id, h);
    if (s < 0) return -1;
    for (int k = 0; k < n; k++)
        if (k != j && ids[k] == id) return -1;
    if (max_entry_variance >= 0.0 && !(e[s].pose.var <= max_entry_variance)) return -1;
    return s;
}

// A counted marker's board entries: obj [4][3] its map-frame corners (float32), img [4][2] its corners, len_f its length as
// fid_pose narrows it, mpose {R 9, t 3} its map pose.
FID_HD void loc_stage_marker(const MapEntry& ent, double len, const float* corners, float* obj, float* img, float* len_f, double* mpose) {
    double o[4][3];
    ba_object_points(len, o);
    ba_map_corners(ent.pose.R, ent.pose.t, o, obj);
    for (int k = 0; k < 8; k++) img[k] = corners[k];
    *len_f = (float)len;
    for (int k = 0; k < 9; k++) mpose[k] = ent.pose.R[k];
    for (int k = 0; k < 3; k++) mpose[9 + k] = ent.pose.t[k];
}

// One frame's localization from its n >= 1 counted markers (obj [4n][3], img [4n][2], mn [4n][2] scratch, len_f [n], mpose
// [n][12] as loc_stage_marker stages them).  camBase: T_camBase (or null); p0 (optional): the LM's start {rvec, tvec}.
// Fills every field of out.
FID_HD void loc_solve(int n, const float* obj, const float* img, double* mn, const Camera& cam, const float* len_f, const double* mpose, double fiducial_len,
                      const Twv* camBase, fid_localization* out, double* p0 = nullptr) {
    const int np = 4 * n;
    memset(out, 0, sizeof(*out));  // the padding too: records compare bit for bit
    out->status = FID_LOC_NO_START;
    out->n_markers = n;
    out->n_points = np;
    out->start = -1;
    out->have_base = camBase != nullptr;
    if (n == 0) {
        out->status = FID_LOC_NONE;
        return;
    }
    double pose[12];
    int start = -1;
    if (!ba_init_frame(n, obj, img, mn, cam, len_f, mpose, pose, &start)) return;
    double p[6];
    rodrigues_m2v(pose, p);
    for (int k = 0; k < 3; k++) p[3 + k] = pose[9 + k];
    if (p0)
        for (int k = 0; k < 6; k++) p0[k] = p[k];
    out->status = FID_LOC_POSE;
    out->start = start;
    out->lm_iters = board_pose_lm(np, obj, img, cam, p);
    out->image_error = board_sq_error(np, obj, img, cam, p, true) / np;
    for (int k = 0; k < 3; k++) {
        out->rvec[k] = p[k];
        out->tvec[k] = p[3 + k];
    }
    // T_mapCam = T_camMap^-1, then T_mapBase = T_mapCam T_camBase (updatePose's composition, map.cpp:284)
    Twv camMap;
    double dRdr[27];
    rodrigues_v2m(p, camMap.R, dRdr);
    for (int k = 0; k < 3; k++) camMap.t[k] = p[3 + k];
    camMap.var = 0.0;
    const Twv mapCam = twv_inverse(camMap);
    const Twv mapX = camBase ? twv_mul(mapCam, *camBase) : mapCam;
    for (int k = 0; k < 3; k++) out->t[k] = mapX.t[k];
    m_to_q(mapX.R, out->q);
    // object_error over the counted markers, in detection order
    double diag = 0.0, depth = 0.0;
    for (int j = 0; j < n; j++) {
        const float* c = img + 8 * j;
        diag += dist2f(c[0], c[1], c[4], c[5]);
        const double* tm = mpose + 12 * j + 9;
        double d2 = 0.0;
        for (int i = 0; i < 3; i++) {
            const double x = camMap.R[3 * i] * tm[0] + camMap.R[3 * i + 1] * tm[1] + camMap.R[3 * i + 2] * tm[2] + camMap.t[i];
            d2 += x * x;
        }
        depth += sqrt(d2);
    }
    out->object_error = (out->image_error / (diag / n)) * ((depth / n) / fiducial_len);
    // covariance: J^T J (upper 21) and sum |e|^2 over every corner at the final pose
    double s[22];
    board_sum<22>(np, [&](int i, double v[22]) {
        const double X[3] = {obj[3 * i], obj[3 * i + 1], obj[3 * i + 2]};
        double uv[2], J[2][6], B[2][3], Jd[2][6];
        project_point(X[0], X[1], X[2], camMap.R, dRdr, p, cam, uv, J);
        const double vx = X[0] - mapX.t[0], vy = X[1] - mapX.t[1], vz = X[2] - mapX.t[2];
        for (int r = 0; r < 2; r++) {
            for (int k = 0; k < 3; k++) B[r][k] = J[r][3] * camMap.R[k] + J[r][4] * camMap.R[3 + k] + J[r][5] * camMap.R[6 + k];  // (dpi/dX_cam) R_cm
            Jd[r][0] = -B[r][0];
            Jd[r][1] = -B[r][1];
            Jd[r][2] = -B[r][2];
            Jd[r][3] = B[r][1] * vz - B[r][2] * vy;  // B [v]x
            Jd[r][4] = B[r][2] * vx - B[r][0] * vz;
            Jd[r][5] = B[r][0] * vy - B[r][1] * vx;
        }
        int o = 0;
        for (int a = 0; a < 6; a++)
            for (int b = a; b < 6; b++) v[o++] = Jd[0][a] * Jd[0][b] + Jd[1][a] * Jd[1][b];
        const double ex = uv[0] - img[2 * i], ey = uv[1] - img[2 * i + 1];
        v[21] = ex * ex + ey * ey;
    }, s);
    out->sigma2 = s[21] / (double)(2 * np - 6);
    double L[21];
    if (!calib_chol6(s, 1.0, L)) return;
    out->cov_ok = 1;
    for (int b = 0; b < 6; b++) {
        double e[6] = {0, 0, 0, 0, 0, 0}, y[6], x[6];
        e[b] = 1.0;
        calib_ro_lsolve6(L, e, y);
        calib_ro_ltsolve6(L, y, x);
        for (int a = 0; a <= b; a++) out->covariance[6 * a + b] = out->covariance[6 * b + a] = out->sigma2 * x[a];
    }
}

}  // namespace fid
