// Candidate ordering and grouping: the float arithmetic of cv::aruco's MarkerCandidateTree /
// filterTooCloseCandidates (OpenCV 4.13 semantics, SURVEY.md A.5), executed by the reference at
// aruco_detect/src/aruco_detect.cpp:350.  All quantities are float32 exactly as in OpenCV
// (Point2f corners, float perimeter, float distances); the library is compiled with --fmad=false.
#pragma once
#include "common.cuh"

namespace fid {

struct QuadF {
    float x[4], y[4];
};

// cv::pointPolygonTest(quad, pt, measureDist=false) > 0 for a float quad (crossing number with OpenCV's edge rules): strictly inside.
FID_HD bool point_strictly_in_quad(const QuadF& q, float px, float py) {
    int counter = 0;
    float vx = q.x[3], vy = q.y[3];
    for (int i = 0; i < 4; i++) {
        const float v0x = vx, v0y = vy;
        vx = q.x[i];
        vy = q.y[i];
        if ((v0y <= py && vy <= py) || (v0y > py && vy > py) || (v0x < px && vx < px)) {
            if (py == vy && (px == vx || (py == v0y && ((v0x <= px && px <= vx) || (vx <= px && px <= v0x))))) return false;  // on the boundary
            continue;
        }
        double dist = (double)(py - v0y) * (vx - v0x) - (double)(px - v0x) * (vy - v0y);
        if (dist == 0) return false;
        if (vy < v0y) dist = -dist;
        counter += dist > 0 ? 1 : 0;
    }
    return (counter & 1) != 0;
}
// checkMarker1InMarker2 of OpenCV 4.13's candidate hierarchy (SURVEY A.5): all four corners of `inner` lie inside `outer`
FID_HD bool quad_inside_quad(const QuadF& inner, const QuadF& outer) {
    for (int k = 0; k < 4; k++)
        if (!point_strictly_in_quad(outer, inner.x[k], inner.y[k])) return false;
    return true;
}

// Raw candidate emitted by the approximation kernel.
struct RawQuad {
    int16_t x[4], y[4];  // approxPolyDP vertex order
    uint32_t n_contour : 24;  // contour length (points)
    uint32_t order_hi : 8;    // scale index  (one word with n_contour: the record stays 28 bytes)
    uint32_t order_lo;   // 0xFFFFFFFF - (2*raster(start)+is_hole): ascending == OpenCV's list order
    uint32_t pts_off;    // the contour's points (findContours order) in the batch point buffer: CORNER_REFINE_CONTOUR fits lines to them
};

// _reorderCandidatesCorners: make the quad clockwise.
FID_HD QuadF quad_clockwise(const RawQuad& r) {
    QuadF q;
    for (int i = 0; i < 4; i++) {
        q.x[i] = (float)r.x[i];
        q.y[i] = (float)r.y[i];
    }
    const double dx1 = q.x[1] - q.x[0], dy1 = q.y[1] - q.y[0];
    const double dx2 = q.x[2] - q.x[0], dy2 = q.y[2] - q.y[0];
    if (dx1 * dy2 - dy1 * dx2 < 0.0) {
        float t = q.x[1];
        q.x[1] = q.x[3];
        q.x[3] = t;
        t = q.y[1];
        q.y[1] = q.y[3];
        q.y[3] = t;
    }
    return q;
}

FID_HD float quad_perimeter(const QuadF& q) {
    float p = 0.f;
    for (int i = 0; i < 4; i++) {
        const float dx = q.x[i] - q.x[(i + 1) & 3], dy = q.y[i] - q.y[(i + 1) & 3];
        p += sqrtf(dx * dx + dy * dy);
    }
    return p;
}

// getAverageDistance: sqrt(min over the 4 cyclic corner alignments of the mean squared distance).
FID_HD float quad_avg_distance(const QuadF& a, const QuadF& b) {
    float best = 3.402823466e+38f;
    for (int fc = 0; fc < 4; fc++) {
        float d = 0.f;
        for (int c = 0; c < 4; c++) {
            const int mc = (c + fc) & 3;
            const float dx = a.x[mc] - b.x[c], dy = a.y[mc] - b.y[c];
            d += dx * dx + dy * dy;
        }
        d /= 4.f;
        best = d < best ? d : best;
    }
    return sqrtf(best);
}

// minDistanceToBorder rule, applied to SELECTED candidates after grouping (see approx_quad.cuh note).
FID_HD bool quad_near_border(const QuadF& q, int W, int H, int min_dist_to_border) {
    const float lo = (float)min_dist_to_border, hx = (float)(W - 1 - min_dist_to_border), hy = (float)(H - 1 - min_dist_to_border);
    for (int j = 0; j < 4; j++)
        if (q.x[j] < lo || q.y[j] < lo || q.x[j] > hx || q.y[j] > hy) return true;
    return false;
}

// getAverageModuleSize
FID_HD float quad_module_size(const QuadF& q, int marker_size, int border_bits) {
    float s = quad_perimeter(q);
    const int modules = marker_size + 2 * border_bits;
    s /= (4.f * (float)modules);
    return s;
}

// Pass 1 (order dependent, serial): the close pairs in row-major order -> groups as linked lists.
// selected[i] = 1 for candidates that are in no group.  Split into init + one call per matrix row so that the device can stage
// a row with a whole warp (one coalesced load) while a single lane applies the sequential rule.
FID_HD void group_pairs_init(int n, uint8_t* selected, int* group_id, int* next_in_group, int* close_count, uint32_t* grouped) {
    for (int i = 0; i < n; i++) {
        selected[i] = 1;
        group_id[i] = -1;
        next_in_group[i] = -1;
        close_count[i] = 0;
    }
    const int n_words = (n + 31) >> 5;
    for (int w = 0; w < n_words; w++) grouped[w] = 0;
}

// OpenCV visits the close pairs (i, j > i) in row-major order: both ungrouped -> new group; one
// grouped -> the other joins it; both grouped -> nothing (groups never merge).  The same marker seen at
// 13 scales gives hundreds of "both grouped" pairs per marker; the `grouped` bit mask skips them a
// word at a time (such a pair changes nothing: selected[] is already 0 for every grouped candidate).
// row(w) = word w of row i of the close-pair matrix; nonempty (optional, 4 words = 128 bits) flags the words of the row that are
// not zero, so that a sparse row costs a few iterations instead of one per word.
template <class Row>
FID_HD void group_pairs_row(int n, int i, const Row& row, const uint32_t* nonempty, int* n_groups, uint8_t* selected, int* group_id, int* next_in_group, int* group_head,
                            int* group_tail, uint32_t* grouped) {
    const int n_words = (n + 31) >> 5;
    for (int w = (i + 1) >> 5; w < n_words; w++) {
        if (nonempty) {  // jump to the next flagged word
            uint32_t m = nonempty[w >> 5] & (0xFFFFFFFFu << (w & 31));
            int q = w >> 5;
            while (!m && ++q < 4) m = nonempty[q];
            if (!m) break;
            w = (q << 5) + fid_ctz(m);
            if (w >= n_words) break;
        }
        uint32_t bits = row(w);
        if (w == ((i + 1) >> 5)) bits &= (i & 31) == 31 ? 0xFFFFFFFFu : ~((2u << (i & 31)) - 1u);  // j > i only
        if (w == n_words - 1 && (n & 31)) bits &= (1u << (n & 31)) - 1u;                            // j < n only
        while (bits) {
            if (group_id[i] >= 0) {
                bits &= ~grouped[w];
                if (!bits) break;
            }
            const int j = (w << 5) + fid_ctz(bits);
            bits &= bits - 1;
            selected[i] = 0;
            selected[j] = 0;
            if (group_id[i] < 0 && group_id[j] < 0) {
                const int g = (*n_groups)++;
                group_id[i] = group_id[j] = g;
                group_head[g] = i;
                next_in_group[i] = j;
                group_tail[g] = j;
                grouped[i >> 5] |= 1u << (i & 31);
                grouped[j >> 5] |= 1u << (j & 31);
            } else if (group_id[i] > -1 && group_id[j] == -1) {
                const int g = group_id[i];
                group_id[j] = g;
                next_in_group[group_tail[g]] = j;
                group_tail[g] = j;
                grouped[j >> 5] |= 1u << (j & 31);
            } else if (group_id[j] > -1 && group_id[i] == -1) {
                const int g = group_id[j];
                group_id[i] = g;
                next_in_group[group_tail[g]] = i;
                group_tail[g] = i;
                grouped[i >> 5] |= 1u << (i & 31);
            }
        }
    }
}

// Returns the number of groups.
template <class CloseWord>
FID_HD int group_pairs(int n, const CloseWord& close_word, uint8_t* selected, int* group_id, int* next_in_group, int* group_head, int* group_tail, int* close_count,
                       uint32_t* grouped) {
    int n_groups = 0;
    group_pairs_init(n, selected, group_id, next_in_group, close_count, grouped);
    struct RowOf {
        const CloseWord& cw;
        int i;
        FID_HD uint32_t operator()(int w) const { return cw(i, w); }
    };
    for (int i = 0; i < n; i++) {
        if (!close_word.row_any(i)) continue;
        group_pairs_row(n, i, RowOf{close_word, i}, nullptr, &n_groups, selected, group_id, next_in_group, group_head, group_tail, grouped);
    }
    return n_groups;
}

// Pass 2 for one group, executed by a lane group (a CUDA warp in k_sort_group, a single lane in tests/hostsim;
// identify.cuh has the Lanes interface): sort the members ascending (largest perimeter first), keep the first,
// collect the "close contours" that differ enough from the running reference -- the lanes test the next
// count() members against the reference at once and the first hit becomes the new reference, which is the
// sequential rule.  members: scratch shared by all groups (2 ints per candidate), *members_used /
// *total_close: reservation counters (atomics on the device).
// SMALLEST_FIRST (detectInvertedMarker, DESIGN.md finding 18 B): the members are sorted descending instead -- the group keeps its
// smallest-perimeter member and collects the close contours from there outward.
template <bool SMALLEST_FIRST = false, class Lanes>
FID_HD void group_finish_lanes(const Lanes& L, int g, const QuadF* quads, int marker_size, int border_bits, float min_group_dist, uint8_t* selected, int* members,
                               int* members_used, const int* next_in_group, const int* group_head, int* close_count, int* close_idx, int* close_off, int* total_close) {
    const int lane = L.lane(), width = L.count();
    int m = 0, base = 0;
    if (lane == 0) {
        for (int k = group_head[g]; k >= 0; k = next_in_group[k]) m++;
        base = L.atomic_add(members_used, 2 * m);  // m members + up to m accepted ids
        int w = 0;
        for (int k = group_head[g]; k >= 0; k = next_in_group[k]) members[base + w++] = k;
    }
    m = L.shfl_i(m, 0);
    base = L.shfl_i(base, 0);
    int* mem = members + base;
    int* acc = mem + m;
    L.sync();
    if (m <= width) {  // rank sort, one member per lane
        const int mine = lane < m ? mem[lane] : 0x7fffffff;
        int rank = 0;
        for (int k = 0; k < m; k++) rank += (SMALLEST_FIRST ? L.shfl_i(mine, k) > mine : L.shfl_i(mine, k) < mine) ? 1 : 0;
        L.sync();
        if (lane < m) mem[rank] = mine;
    } else if (lane == 0) {
        for (int x = 1; x < m; x++) {  // insertion sort (rare: more members than lanes)
            const int v = mem[x];
            int b = x - 1;
            while (b >= 0 && (SMALLEST_FIRST ? mem[b] < v : mem[b] > v)) {
                mem[b + 1] = mem[b];
                b--;
            }
            mem[b + 1] = v;
        }
    }
    L.sync();
    const int lead = mem[0];
    int cur = lead, n_acc = 0, pos = 1;
    while (pos < m) {
        const int x = pos + lane;
        bool ok = false;
        if (x < m) {
            const int id = mem[x];
            const QuadF q = quads[id];
            ok = quad_avg_distance(q, quads[cur]) > min_group_dist * quad_module_size(q, marker_size, border_bits);
        }
        const uint32_t hits = L.ballot(ok);
        if (!hits) {
            pos += width;
            continue;
        }
        const int first = pos + fid_ctz(hits);
        cur = mem[first];
        if (lane == 0) acc[n_acc] = cur;
        n_acc++;
        pos = first + 1;
    }
    L.sync();
    int off = 0;
    if (lane == 0) {
        off = L.atomic_add(total_close, n_acc);
        selected[lead] = 1;
        close_off[lead] = off;
        close_count[lead] = n_acc;
    }
    off = L.shfl_i(off, 0);
    for (int k = lane; k < n_acc; k += width) close_idx[off + k] = acc[k];
}

// Both passes, serial (CPU harness).  `close_word(i, w)` returns bits [32w, 32w+32) of row i of the pair
// predicate avgDist(i,j) < perimeter[j] * minMarkerDistanceRate (upper triangle, j > i), `close_word.row_any(i)`
// whether row i has any bit.  Outputs: selected[i] and, for group leaders, the list of close contours
// (indices) in close_idx[close_off[i] .. close_off[i] + close_count[i]).  SMALLEST_FIRST: as group_finish_lanes.
template <bool SMALLEST_FIRST = false, class Lanes, class CloseWord>
FID_HD void group_candidates(const Lanes& L, int n, const QuadF* quads, int marker_size, int border_bits, float min_group_dist, const CloseWord& close_word, uint8_t* selected,
                             int* group_id,        // [n]
                             int* group_members,   // [2n]  scratch
                             int* next_in_group,   // [n]   linked list
                             int* group_head,      // [n]   head per group
                             int* group_tail,      // [n]
                             int* close_count,     // [n]   number of close contours per candidate
                             int* close_idx,       // [n]   flat storage
                             int* close_off,       // [n+1]
                             uint32_t* grouped)    // [(n+31)/32] scratch
{
    const int n_groups = group_pairs(n, close_word, selected, group_id, next_in_group, group_head, group_tail, close_count, grouped);
    int total_close = 0, members_used = 0;
    for (int g = 0; g < n_groups; g++)
        group_finish_lanes<SMALLEST_FIRST>(L, g, quads, marker_size, border_bits, min_group_dist, selected, group_members, &members_used, next_in_group, group_head, close_count, close_idx, close_off,
                           &total_close);
}

}  // namespace fid
