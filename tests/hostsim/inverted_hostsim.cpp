// CPU harness of detection with detectInvertedMarker (DESIGN.md finding 18).  TEST INFRASTRUCTURE ONLY.  Compiled with g++ by
// tests/inverted_oracle.py into a shared object of its own in a temporary directory; it is not linked into libfiducials_b200.so.
// It compiles the same headers as hs_detect (it includes hostsim.cpp for the candidate stage) and replays, with one lane, what the
// device runs: grouping (group_candidates<SMALLEST_FIRST>), the identification kernels (identify_candidate<CONF, INV>, with the
// confidence of marker_confidence), the candidate hierarchy of k_finish, and CORNER_REFINE_CONTOUR / cornerSubPix.
#include "hostsim.cpp"

#include "../../fiducials_b200/csrc/candidate_tree.cuh"

extern "C" {

// One candidate quad (x0,y0..x3,y3, clockwise) identified with both polarities tried when `inverted` is set: out = id, rotation,
// polarity (1 = read inverted); *conf = its confidence.  prm as hs_detect_inv.  Returns 0, or -2 for bad parameters.
int hs_identify_inv(const uint8_t* gray, int W, int H, const float* quad, const double* prm, int inverted, int32_t* out, float* conf);

// gray [H][W], planes [n_scales][H][W] of the reference parameters.  prm = dictionary, cornerRefinementMethod (0, 1, 2),
// markerBorderBits, perspectiveRemovePixelPerCell, perspectiveRemoveIgnoredMarginPerCell, errorCorrectionRate,
// maxErroneousBitsInBorderRate; the other parameters are the reference's.  inverted = detectInvertedMarker.  ids [max_out],
// corners [max_out][8], conf [max_out], polarity [max_out] (1 = white marker).  Returns the number of markers, -1 if they do not
// fit, -2 for bad parameters.
int hs_detect_inv(const uint8_t* gray, const uint8_t* planes, int W, int H, const double* prm, int inverted, int32_t* ids, float* corners, float* conf, int32_t* polarity,
                  int max_out);

}  // extern "C"

namespace {

int inv_params(const double* prm, DevParams* P) {
    fid_params fp;
    default_params(&fp);
    fp.dictionary = (int)prm[0];
    fp.cornerRefinementMethod = (int)prm[1];
    fp.markerBorderBits = (int)prm[2];
    fp.perspectiveRemovePixelPerCell = (int)prm[3];
    fp.perspectiveRemoveIgnoredMarginPerCell = prm[4];
    fp.errorCorrectionRate = prm[5];
    fp.maxErroneousBitsInBorderRate = prm[6];
    return make_dev_params(fp, P) == FID_OK ? 0 : -2;
}

IdentifyResult identify(bool inverted, const GrayPlane& g, int W, int H, const QuadF& q, const DevParams& P, const unsigned long long* dict, uint8_t* img, int* hist) {
    return inverted ? identify_candidate<true, true>(SerialLanes(), g, W, H, q, P, dict, img, hist) : identify_candidate<true>(SerialLanes(), g, W, H, q, P, dict, img, hist);
}

}  // namespace

int hs_identify_inv(const uint8_t* gray, int W, int H, const float* quad, const double* prm, int inverted, int32_t* out, float* conf) {
    DevParams P;
    if (inv_params(prm, &P)) return -2;
    std::vector<unsigned long long> dict;
    pack_dictionary(P, &dict);
    QuadF q;
    for (int c = 0; c < 4; c++) {
        q.x[c] = quad[2 * c];
        q.y[c] = quad[2 * c + 1];
    }
    std::vector<uint8_t> img(FID_MAX_WARP_SIDE_SQ);
    int hist[256];
    const IdentifyResult r = identify(inverted != 0, GrayPlane{gray, (size_t)W}, W, H, q, P, dict.data(), img.data(), hist);
    out[0] = r.id;
    out[1] = r.rotation;
    out[2] = r.inverted ? 1 : 0;
    *conf = r.id >= 0 ? marker_confidence(hist, P, dict[(size_t)r.id * 4 + r.rotation]) : 0.0f;
    return 0;
}

int hs_detect_inv(const uint8_t* gray, const uint8_t* planes, int W, int H, const double* prm, int inverted, int32_t* ids, float* corners, float* conf, int32_t* polarity,
                  int max_out) {
    DevParams P;
    if (inv_params(prm, &P)) return -2;
    std::vector<RawQuad> raw;
    std::vector<Pt16> contour_pts;
    raw_candidates(planes, W, H, P, raw, &contour_pts);
    const int n = (int)raw.size();
    std::vector<QuadF> q(n);
    std::vector<float> per(n);
    std::vector<int> order(n);
    for (int i = 0; i < n; i++) {
        q[i] = quad_clockwise(raw[i]);
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
    } close_word{&sq, &sper, n, (float)P.min_marker_dist_rate};
    std::vector<uint8_t> selected(n);
    std::vector<int> gid(n), gmem(2 * (size_t)n + 2), nxt(n), ghead(n), gtail(n), ccount(n), cidx(n), coff(n + 1);
    std::vector<uint32_t> grouped_bits((size_t)(n + 31) / 32 + 1);
    if (inverted)
        group_candidates<true>(SerialLanes(), n, sq.data(), P.marker_size, P.marker_border_bits, (float)P.min_group_dist, close_word, selected.data(), gid.data(), gmem.data(),
                               nxt.data(), ghead.data(), gtail.data(), ccount.data(), cidx.data(), coff.data(), grouped_bits.data());
    else
        group_candidates(SerialLanes(), n, sq.data(), P.marker_size, P.marker_border_bits, (float)P.min_group_dist, close_word, selected.data(), gid.data(), gmem.data(),
                         nxt.data(), ghead.data(), gtail.data(), ccount.data(), cidx.data(), coff.data(), grouped_bits.data());
    std::vector<int> sel;
    for (int i = 0; i < n; i++)
        if (selected[i] && !quad_near_border(sq[i], W, H, P.min_dist_to_border)) sel.push_back(i);
    const int ns = std::min((int)sel.size(), 512);  // FID_MAX_SEL
    std::vector<unsigned long long> dict;
    pack_dictionary(P, &dict);
    std::vector<uint8_t> img(FID_MAX_WARP_SIDE_SQ);
    int hist[256];
    const GrayPlane gp{gray, (size_t)W};
    // identification: the selected quad, then its close contours in order; the confidence from the attempt that decoded
    std::vector<int> cand_id(ns), cand_rot(ns), cand_use(ns), cand_pol(ns);
    std::vector<float> cand_conf(ns);
    for (int k = 0; k < ns; k++) {
        const int i = sel[k];
        int use = i;
        IdentifyResult r = identify(inverted != 0, gp, W, H, sq[i], P, dict.data(), img.data(), hist);
        for (int c = 0; c < ccount[i] && r.id < 0; c++) {
            use = cidx[coff[i] + c];
            r = identify(inverted != 0, gp, W, H, sq[use], P, dict.data(), img.data(), hist);
        }
        cand_id[k] = r.id;
        cand_rot[k] = r.rotation;
        cand_use[k] = use;
        cand_pol[k] = r.inverted ? 1 : 0;
        if (r.id >= 0) cand_conf[k] = marker_confidence(hist, P, dict[(size_t)r.id * 4 + r.rotation]);
    }
    // the candidate hierarchy, as k_finish runs it
    std::vector<short> parent(ns), depth(ns, 0);
    std::vector<unsigned char> was(ns, 0);
    for (int i = 0; i < ns; i++) parent[i] = (short)tree_parent(sq[sel[i]], i, [&](int j) { return sq[sel[j]]; });
    tree_levels(ns, parent.data(), depth.data(), was.data(), [&](int v) { return cand_id[v] >= 0; });
    float mask[121];
    std::vector<float> patch(13 * 13);
    int n_out = 0;
    for (int k = 0; k < ns; k++) {
        if (cand_id[k] < 0 || !(was[k] & 2)) continue;
        if (n_out >= max_out) return -1;
        const QuadF& use = sq[cand_use[k]];
        float cx[4], cy[4];
        for (int c = 0; c < 4; c++) {  // correctCornerPosition
            cx[c] = use.x[(c + 4 - cand_rot[k]) & 3];
            cy[c] = use.y[(c + 4 - cand_rot[k]) & 3];
        }
        if (P.corner_refine == 2) {
            const RawQuad& rw = raw[order[cand_use[k]]];
            refine_candidate_lines_serial(contour_pts.data() + rw.pts_off, rw.n_contour, cx, cy);
        } else if (P.corner_refine == 1) {
            QuadF rq;
            for (int c = 0; c < 4; c++) {
                rq.x[c] = cx[c];
                rq.y[c] = cy[c];
            }
            const float module = quad_module_size(rq, P.marker_size, P.marker_border_bits);
            int win = (int)nearbyintf((float)P.rel_refine_win * module);
            win = win < 1 ? 1 : win;
            win = win < P.refine_win ? win : P.refine_win;
            subpix_mask(win, mask);
            for (int c = 0; c < 4; c++)
                corner_subpix(gp, W, H, &cx[c], &cy[c], win, mask, P.refine_max_iter, P.refine_min_acc * P.refine_min_acc, patch.data());
        }
        ids[n_out] = cand_id[k];
        conf[n_out] = cand_conf[k];
        polarity[n_out] = cand_pol[k];
        for (int c = 0; c < 4; c++) {
            corners[n_out * 8 + 2 * c] = cx[c];
            corners[n_out * 8 + 2 * c + 1] = cy[c];
        }
        n_out++;
    }
    return n_out;
}
