// CPU harness of detection with useAruco3Detection (fiducials_b200/csrc/aruco3.cuh, DESIGN.md finding 16).  TEST INFRASTRUCTURE
// ONLY.  Compiled with g++ by tests/aruco3_oracle.py into a shared object of its own in a temporary directory; it is not linked into
// libfiducials_b200.so.  It compiles the same headers as hs_detect (it includes hostsim.cpp for the candidate stage) and replays,
// with one lane, what the device runs in the mode: the planes (k_a3_pyr_down, k_a3_resize), the candidate stage on the
// segmentation plane with the minimum contour length 4 * minSide, grouping, identification on each candidate's pyramid level, the
// candidate hierarchy of k_finish, and the corner stage of k_a3_corners.
#include "hostsim.cpp"

#include "../../fiducials_b200/csrc/aruco3.cuh"
#include "../../fiducials_b200/csrc/candidate_tree.cuh"

namespace {

struct A3Planes {
    A3Geom g;
    std::vector<std::vector<uint8_t>> lv;  // level l: lv[l].size() == W * H (pitch W; level 0 is the gray plane)
    std::vector<uint8_t> seg;
};

bool build_planes(const uint8_t* gray, int W, int H, int min_side, double ratio, A3Planes& p) {
    if (!a3_geometry(W, H, min_side, ratio, &p.g)) return false;
    p.lv.assign(p.g.n_levels, {});
    p.lv[0].assign(gray, gray + (size_t)W * H);
    for (int l = 1; l < p.g.n_levels; l++) {
        const int sw = p.g.lv[l - 1].W, sh = p.g.lv[l - 1].H, w = p.g.lv[l].W, h = p.g.lv[l].H;
        p.lv[l].resize((size_t)w * h);
        const GrayPlane src{p.lv[l - 1].data(), (size_t)sw};
        for (int y = 0; y < h; y++)
            for (int x = 0; x < w; x++) p.lv[l][(size_t)y * w + x] = (uint8_t)a3_pyr_down_at(src, sw, sh, x, y);
    }
    const int sw = p.g.seg_w, sh = p.g.seg_h;
    p.seg.resize((size_t)sw * sh);
    const double scx = 1.0 / ((double)sw / W), scy = 1.0 / ((double)sh / H);
    const GrayPlane src{gray, (size_t)W};
    for (int y = 0; y < sh; y++)
        for (int x = 0; x < sw; x++) p.seg[(size_t)y * sw + x] = (uint8_t)a3_resize_at(src, W, H, scx, scy, x, y);
    return true;
}

}  // namespace

extern "C" {

// info: seg_w, seg_h, n_levels, closest.  seg [seg_h][seg_w]; pyr: levels 1.. concatenated, each W x H.  Returns 0, or -2 for a
// pyramid deeper than FID_ARUCO3_MAX_LEVELS.
int hs_a3_planes(const uint8_t* gray, int W, int H, int min_side, double ratio, int32_t* info, uint8_t* seg, uint8_t* pyr) {
    A3Planes p;
    if (!build_planes(gray, W, H, min_side, ratio, p)) return -2;
    info[0] = p.g.seg_w;
    info[1] = p.g.seg_h;
    info[2] = p.g.n_levels;
    info[3] = p.g.closest;
    if (seg) memcpy(seg, p.seg.data(), p.seg.size());
    if (pyr)
        for (int l = 1; l < p.g.n_levels; l++) memcpy(pyr + p.g.lv[l].off, p.lv[l].data(), p.lv[l].size());
    return 0;
}

// Pyramid level of a contour of length n (a3_level_for).
int hs_a3_level_for(int W, int H, int min_side, double ratio, int n) {
    A3Geom g;
    if (!a3_geometry(W, H, min_side, ratio, &g)) return -2;
    return a3_level_for(g, n);
}

// gray [H][W]; seg_planes [n_scales][seg_h][seg_w]: the reference threshold planes of the segmentation plane.  ids [max_out],
// corners [max_out][8] at full resolution.  Returns the number of markers, -1 if they do not fit, -2 for bad parameters.
int hs_detect_aruco3(const uint8_t* gray, int W, int H, const uint8_t* seg_planes, int dict_id, int min_side, double ratio, int32_t* ids, float* corners,
                     int max_out) {
    A3Planes pl;
    if (!build_planes(gray, W, H, min_side, ratio, pl)) return -2;
    const A3Geom& g = pl.g;
    const int sw = g.seg_w, sh = g.seg_h;
    fid_params fp;
    default_params(&fp);
    fp.dictionary = dict_id;
    DevParams P;
    if (make_dev_params(fp, &P) != FID_OK) return -2;
    // raw_candidates takes the minimum contour length as (int)(rate * max side): a rate half a pixel above 4 * minSide gives it
    DevParams Pc = P;
    Pc.min_perimeter_rate = (4.0 * min_side + 0.5) / (sw > sh ? sw : sh);
    std::vector<RawQuad> raw;
    std::vector<Pt16> contour_pts;
    raw_candidates(seg_planes, sw, sh, Pc, raw, &contour_pts);
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
    group_candidates(SerialLanes(), n, sq.data(), P.marker_size, P.marker_border_bits, (float)P.min_group_dist, close_word, selected.data(), gid.data(), gmem.data(),
                     nxt.data(), ghead.data(), gtail.data(), ccount.data(), cidx.data(), coff.data(), grouped_bits.data());
    std::vector<int> sel;
    for (int i = 0; i < n; i++)
        if (selected[i] && !quad_near_border(sq[i], sw, sh, P.min_dist_to_border)) sel.push_back(i);
    const int ns = std::min((int)sel.size(), 512);  // FID_MAX_SEL
    std::vector<unsigned long long> dict;
    pack_dictionary(P, &dict);
    const SerialLanes L;
    std::vector<uint8_t> img(FID_MAX_WARP_SIDE_SQ);
    int hist[256];
    // identification on the selected candidate's pyramid level, for it and its close contours alike
    std::vector<int> cand_id(ns), cand_rot(ns), cand_use(ns);
    for (int k = 0; k < ns; k++) {
        const int i = sel[k];
        const int level = a3_level_for(g, raw[order[i]].n_contour);
        const float s = a3_level_scale(g, level);
        const GrayPlane im{pl.lv[level].data(), (size_t)g.lv[level].W};
        auto attempt = [&](const QuadF& qq) {
            QuadF t;
            for (int c = 0; c < 4; c++) {
                t.x[c] = qq.x[c] * s;
                t.y[c] = qq.y[c] * s;
            }
            return identify_candidate(L, im, g.lv[level].W, g.lv[level].H, t, P, dict.data(), img.data(), hist);
        };
        int use = i;
        IdentifyResult r = attempt(sq[i]);
        for (int c = 0; c < ccount[i] && r.id < 0; c++) {
            use = cidx[coff[i] + c];
            r = attempt(sq[use]);
        }
        cand_id[k] = r.id;
        cand_rot[k] = r.rotation;
        cand_use[k] = use;
    }
    std::vector<short> parent(ns), depth(ns, 0);
    std::vector<unsigned char> was(ns, 0);
    for (int i = 0; i < ns; i++) parent[i] = (short)tree_parent(sq[sel[i]], i, [&](int j) { return sq[sel[j]]; });
    tree_levels(ns, parent.data(), depth.data(), was.data(), [&](int v) { return cand_id[v] >= 0; });
    float mask3[49], mask5[121];
    subpix_mask(3, mask3);
    subpix_mask(5, mask5);
    std::vector<float> patch(13 * 13);
    auto plane = [&](int l) { return GrayPlane{pl.lv[l].data(), (size_t)g.lv[l].W}; };
    auto mask = [&](int win) -> const float* { return win == 5 ? mask5 : mask3; };
    int n_out = 0;
    for (int k = 0; k < ns; k++) {
        if (cand_id[k] < 0 || !(was[k] & 2)) continue;
        if (n_out >= max_out) return -1;
        const QuadF& use = sq[cand_use[k]];
        for (int c = 0; c < 4; c++) {  // correctCornerPosition, then findCornerInPyrImage
            float x = use.x[(c + 4 - cand_rot[k]) & 3], y = use.y[(c + 4 - cand_rot[k]) & 3];
            a3_upsample_corner(g, plane, mask, P.refine_max_iter, P.refine_min_acc * P.refine_min_acc, &x, &y, patch.data());
            corners[n_out * 8 + 2 * c] = x;
            corners[n_out * 8 + 2 * c + 1] = y;
        }
        ids[n_out] = cand_id[k];
        n_out++;
    }
    return n_out;
}

}  // extern "C"
