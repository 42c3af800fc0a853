// CPU harness for fiducials_b200/csrc/map_localize.cuh (fid_map_localize).  TEST INFRASTRUCTURE ONLY.  Compiled with g++ by
// tests/test_hostsim_map_localize.py into a shared object of its own in a temporary directory; it is not linked into
// libfiducials_b200.so.  hs_map_localize runs each frame as k_map_localize does, with the detections matched one after another
// (the device compacts them with a ballot prefix in the same order) and the map searched linearly (the device's hash gives the
// same slots).
#include "../../fiducials_b200/csrc/map_localize.cuh"

#include <vector>

using namespace fid;

extern "C" {

// Map: slot_ids [n_slots], var [n_slots], poses [n_slots][12] (R row-major, t).  Frames: counts [n_frames], ids
// [n_frames][max_markers], corners [n_frames][max_markers][8].  cam_base: x y z qx qy qz qw of T_camBase, or null.  Outputs:
// out [n_frames], p0 [n_frames][6] the LM's start (rvec, tvec; 0 without one), used [n_frames][max_markers] the counted detections'
// indices in order (-1 past them).
void hs_map_localize(int n_slots, const int32_t* slot_ids, const double* var, const double* poses, int n_frames, const int32_t* counts, const int32_t* ids,
                     const float* corners, int max_markers, const double* K, const double* D, double fiducial_len, int n_override, const int32_t* override_ids,
                     const double* override_lens, double max_entry_variance, const double* cam_base, fid_localization* out, double* p0, int32_t* used) {
    const Camera cam{K[0], K[4], K[2], K[5], D[0], D[1], D[2], D[3], D[4]};
    std::vector<MapEntry> e(n_slots);
    for (int s = 0; s < n_slots; s++) {
        e[s].id = slot_ids[s];
        e[s].num_obs = 0;
        for (int k = 0; k < 9; k++) e[s].pose.R[k] = poses[12 * s + k];
        for (int k = 0; k < 3; k++) e[s].pose.t[k] = poses[12 * s + 9 + k];
        e[s].pose.var = var[s];
    }
    MapState st{};
    st.n = n_slots;
    Twv camBase{};
    if (cam_base) {
        q_to_m(cam_base + 3, camBase.R);
        for (int k = 0; k < 3; k++) camBase.t[k] = cam_base[k];
    }
    const int mm = max_markers;
    std::vector<float> obj((size_t)12 * mm), img((size_t)8 * mm), len_f(mm);
    std::vector<double> mn((size_t)8 * mm), mpose((size_t)12 * mm);
    for (int f = 0; f < n_frames; f++) {
        const int n = counts[f];
        const int32_t* fid = ids + (size_t)f * mm;
        int k = 0;
        for (int j = 0; j < mm; j++) used[(size_t)f * mm + j] = -1;
        for (int j = 0; j < n; j++) {
            const int s = loc_slot(st, e.data(), nullptr, n, fid, j, max_entry_variance);
            if (s < 0) continue;
            loc_stage_marker(e[s], ba_marker_len(fid[j], fiducial_len, n_override, override_ids, override_lens), corners + (size_t)8 * (f * mm + j), &obj[12 * k],
                             &img[8 * k], &len_f[k], &mpose[12 * k]);
            used[(size_t)f * mm + k] = j;
            k++;
        }
        for (int q = 0; q < 6; q++) p0[6 * f + q] = 0.0;
        loc_solve(k, obj.data(), img.data(), mn.data(), cam, len_f.data(), mpose.data(), fiducial_len, cam_base ? &camBase : nullptr, out + f, p0 + 6 * f);
    }
}

}  // extern "C"
