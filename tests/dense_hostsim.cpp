// CPU harness of the candidate counts of dense frames (tests/test_hostsim_dense.py).  TEST INFRASTRUCTURE ONLY.  Compiled with g++
// by tests/test_hostsim_dense.py into a shared object of its own in a temporary directory; it is not linked into
// libfiducials_b200.so.  It compiles the same headers as hs_detect (it includes hostsim.cpp) and replays hs_detect's chain --
// candidate stage, descending-perimeter sort, grouping, border rule, identification -- with the threshold windows and the minimum
// perimeter rate of the caller instead of the reference's, and without a cap on the marker count, so that frames past the device's
// per-frame capacities can be counted.
#include "hostsim/hostsim.cpp"

extern "C" {

// gray [H][W], planes [n_scales][H][W] of the windows win_min..win_max step win_step.  ids [max_out] in OpenCV's order.
// stats[0] = raw quad candidates, stats[1] = selected candidates (after grouping and the border rule).  Returns the number of
// markers, -1 if they do not fit in max_out, -2 for bad parameters.
int hs_dense_counts(const uint8_t* gray, const uint8_t* planes, int W, int H, int dict_id, int win_min, int win_max, int win_step, double min_perimeter_rate,
                    int32_t* ids, int max_out, int32_t* stats) {
    fid_params fp;
    default_params(&fp);
    fp.dictionary = dict_id;
    fp.adaptiveThreshWinSizeMin = win_min;
    fp.adaptiveThreshWinSizeMax = win_max;
    fp.adaptiveThreshWinSizeStep = win_step;
    fp.minMarkerPerimeterRate = min_perimeter_rate;
    DevParams P;
    if (make_dev_params(fp, &P) != FID_OK) return -2;
    std::vector<RawQuad> raw;
    raw_candidates(planes, W, H, P, raw);
    const int n = (int)raw.size();
    std::vector<QuadF> q(n), sq(n);
    std::vector<float> per(n), sper(n);
    std::vector<int> order(n);
    for (int i = 0; i < n; i++) {
        q[i] = quad_clockwise(raw[i]);
        per[i] = quad_perimeter(q[i]);
        order[i] = i;
    }
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return per[a] > per[b]; });
    for (int i = 0; i < n; i++) {
        sq[i] = q[order[i]];
        sper[i] = per[order[i]];
    }
    std::vector<uint8_t> selected(n);
    std::vector<int> gid(n), gmem(2 * (size_t)n + 2), nxt(n), ghead(n), gtail(n), ccount(n), cidx(n), coff(n + 1);
    std::vector<uint32_t> grouped_bits((size_t)(n + 31) / 32 + 1);
    struct CloseWord {
        const std::vector<QuadF>* sq;
        const std::vector<float>* sper;
        int n;
        float rate;
        uint32_t operator()(int i, int w) const {
            uint32_t bits = 0;
            for (int b = 0; b < 32; b++) {
                const int j = 32 * w + b;
                if (j > i && j < n && quad_avg_distance((*sq)[i], (*sq)[j]) < (*sper)[j] * rate) bits |= 1u << b;
            }
            return bits;
        }
        bool row_any(int) const { return true; }
    } close_word{&sq, &sper, n, (float)P.min_marker_dist_rate};
    group_candidates(SerialLanes(), n, sq.data(), P.marker_size, P.marker_border_bits, (float)P.min_group_dist, close_word, selected.data(), gid.data(), gmem.data(),
                     nxt.data(), ghead.data(), gtail.data(), ccount.data(), cidx.data(), coff.data(), grouped_bits.data());
    std::vector<unsigned long long> dict;
    pack_dictionary(P, &dict);
    std::vector<uint8_t> img(64 * 64);
    int hist[256];
    int n_out = 0, n_sel = 0;
    for (int i = 0; i < n; i++) {
        if (!selected[i] || quad_near_border(sq[i], W, H, P.min_dist_to_border)) continue;
        n_sel++;
        IdentifyResult r = identify_candidate(SerialLanes(), GrayPlane{gray, (size_t)W}, W, H, sq[i], P, dict.data(), img.data(), hist);
        for (int k = 0; r.id < 0 && k < ccount[i]; k++)
            r = identify_candidate(SerialLanes(), GrayPlane{gray, (size_t)W}, W, H, sq[cidx[coff[i] + k]], P, dict.data(), img.data(), hist);
        if (r.id < 0) continue;
        if (n_out >= max_out) return -1;
        ids[n_out++] = r.id;
    }
    stats[0] = n;
    stats[1] = n_sel;
    return n_out;
}

}  // extern "C"
