// CPU harness for fiducials_b200/csrc/candidate_tree.cuh (the OpenCV 4.13 candidate hierarchy): detectMarkers' ids and
// rejectedImgPoints on the host.  TEST INFRASTRUCTURE ONLY.  Compiled with g++ by tests/test_hostsim_rejected.py into a shared object
// of its own in a temporary directory; it is not linked into libfiducials_b200.so.  hs_rejected takes the raw quad candidates of
// the host candidate stage (tests/hostsim/hostsim.cpp, hs_candidates) and replays what k_sort_group, the identification kernels,
// k_finish and k_rejected do after it, with one lane.
#include <algorithm>
#include <vector>

#include "../../fiducials_b200/csrc/candidate_tree.cuh"
#include "../../fiducials_b200/csrc/identify.cuh"
#include "../../fiducials_b200/csrc/params_host.h"
#include "../../fiducials_b200/csrc/quad_group.cuh"

using namespace fid;

extern "C" {

// raw [n_raw][8]: the candidates' integer vertices in the candidate stage's order.  ids [max_ids]: the markers in output order
// (before corner refinement); rej [max_rej][8]: the rejected list.  Returns the number of rejected candidates (*n_ids the markers),
// -1 if a list does not fit, -2 for bad parameters.
int hs_rejected(const uint8_t* gray, int W, int H, int dict_id, int n_raw, const int32_t* raw, int32_t* ids, int max_ids, int* n_ids, float* rej, int max_rej) {
    fid_params fp;
    default_params(&fp);
    fp.dictionary = dict_id;
    DevParams P;
    if (make_dev_params(fp, &P) != FID_OK) return -2;
    const int n = n_raw;
    // clockwise quads, stable sort by descending float perimeter (k_sort_group)
    std::vector<QuadF> q(n);
    std::vector<float> per(n);
    std::vector<int> order(n);
    for (int i = 0; i < n; i++) {
        RawQuad r{};
        for (int k = 0; k < 4; k++) {
            r.x[k] = (int16_t)raw[i * 8 + 2 * k];
            r.y[k] = (int16_t)raw[i * 8 + 2 * k + 1];
        }
        q[i] = quad_clockwise(r);
        per[i] = quad_perimeter(q[i]);
        order[i] = i;
    }
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return per[a] > per[b]; });
    std::vector<QuadF> sq(n);
    std::vector<float> sper(n);
    for (int i = 0; i < n; i++) {
        sq[i] = q[order[i]];
        sper[i] = per[order[i]];
    }
    std::vector<uint8_t> selected(n);
    std::vector<int> gid(n), gmem(2 * (size_t)n + 2), nxt(n), ghead(n), gtail(n), ccount(n), cidx(n), coff(n + 1);
    std::vector<uint32_t> grouped_bits((size_t)(n + 31) / 32 + 1);
    const float rate = (float)P.min_marker_dist_rate;
    struct CloseWordHost {
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
    } close_word{&sq, &sper, n, rate};
    group_candidates(SerialLanes(), n, sq.data(), P.marker_size, P.marker_border_bits, (float)P.min_group_dist, close_word, selected.data(), gid.data(), gmem.data(), nxt.data(),
                     ghead.data(), gtail.data(), ccount.data(), cidx.data(), coff.data(), grouped_bits.data());
    // the selected candidates that pass the border rule, in order, and their identification (first attempt, then the close contours)
    std::vector<int> sel;
    for (int i = 0; i < n; i++)
        if (selected[i] && !quad_near_border(sq[i], W, H, P.min_dist_to_border)) sel.push_back(i);
    const int ns = std::min((int)sel.size(), 512);  // FID_MAX_SEL
    std::vector<unsigned long long> dict;
    pack_dictionary(P, &dict);
    const SerialLanes L;
    std::vector<uint8_t> img(FID_MAX_WARP_SIDE_SQ);
    int hist[256];
    std::vector<int> cand_id(ns);
    for (int k = 0; k < ns; k++) {
        const int i = sel[k];
        IdentifyResult r = identify_candidate(L, GrayPlane{gray, (size_t)W}, W, H, sq[i], P, dict.data(), img.data(), hist);
        for (int c = 0; c < ccount[i] && r.id < 0; c++)
            r = identify_candidate(L, GrayPlane{gray, (size_t)W}, W, H, sq[cidx[coff[i] + c]], P, dict.data(), img.data(), hist);
        cand_id[k] = r.id;
    }
    // the hierarchy, as k_finish and k_rejected run it
    std::vector<short> parent(ns), depth(ns, 0);
    std::vector<unsigned char> was(ns, 0);
    for (int i = 0; i < ns; i++) parent[i] = (short)tree_parent(sq[sel[i]], i, [&](int j) { return sq[sel[j]]; });
    tree_levels(ns, parent.data(), depth.data(), was.data(), [&](int v) { return cand_id[v] >= 0; });
    int ni = 0, nr = 0;
    for (int k = 0; k < ns; k++) {
        if (cand_id[k] >= 0 && (was[k] & 2)) {
            if (ni >= max_ids) return -1;
            ids[ni++] = cand_id[k];
            continue;
        }
        if (nr >= max_rej) return -1;
        for (int c = 0; c < 4; c++) {
            rej[nr * 8 + 2 * c] = sq[sel[k]].x[c];
            rej[nr * 8 + 2 * c + 1] = sq[sel[k]].y[c];
        }
        nr++;
    }
    *n_ids = ni;
    return nr;
}

}  // extern "C"
