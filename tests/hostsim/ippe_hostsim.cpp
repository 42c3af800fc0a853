// CPU harness for fiducials_b200/csrc/ippe.cuh (both planar pose hypotheses of a square marker).  TEST INFRASTRUCTURE ONLY.
// Compiled with g++ by tests/test_hostsim_ippe.py into a shared object of its own in a temporary directory, from the same header
// the CUDA kernel k_pose_hypotheses is built from; it is not linked into libfiducials_b200.so.
#include "../../fiducials_b200/csrc/pnp.cuh"
#include "../../fiducials_b200/csrc/ippe.cuh"

using namespace fid;

extern "C" {

// Both IPPE_SQUARE hypotheses of n markers, next to the ITERATIVE pose of each (solve_marker_pose, for iterative_match);
// out: n x 24 doubles (n match rvec0 rvec1 tvec0 tvec1 rms0 rms1 solver_err0 solver_err1 iterative_rvec, pad)
void hs_pose_hypotheses(int n, const float* corners, const double* K, const double* D, const float* lens, double* out) {
    Camera cam = {K[0], K[4], K[2], K[5], D[0], D[1], D[2], D[3], D[4]};
    for (int i = 0; i < n; i++) {
        PoseOut po;
        solve_marker_pose(corners + 8 * i, cam, lens[i], (double)lens[i], &po);
        PoseHypOut ho;
        solve_marker_hypotheses(corners + 8 * i, cam, lens[i], po.rvec, &ho);
        double* o = out + 24 * i;
        o[0] = ho.n;
        o[1] = ho.iterative_match;
        for (int s = 0; s < 2; s++)
            for (int k = 0; k < 3; k++) {
                o[2 + 3 * s + k] = ho.rvec[s][k];
                o[8 + 3 * s + k] = ho.tvec[s][k];
            }
        o[14] = ho.rms[0];
        o[15] = ho.rms[1];
        o[16] = ho.solver_err[0];
        o[17] = ho.solver_err[1];
        for (int k = 0; k < 3; k++) o[18 + k] = po.rvec[k];
    }
}

}  // extern "C"
