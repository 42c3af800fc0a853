// Mark-free border following on an immutable neighbour-mask plane.
//
// Replaces the findContours(RETR_LIST, CHAIN_APPROX_NONE) pass that cv::aruco::detectMarkers
// (called at aruco_detect/src/aruco_detect.cpp:350) runs on each of the 13 threshold planes.
// OpenCV's Suzuki-Abe scan is sequential (it marks visited pixels); here every border is found
// independently (SURVEY.md A.3b):
//
//  * the walk reads the bit-packed threshold plane directly (halo tiles, below): per step the 3x3
//    neighbourhood of the current pixel indexes a table; conceptually it is an 8-bit occupancy mask
//    (bit k set <=> neighbour in direction k is foreground; pixels outside the image are
//    background, which is OpenCV 4.13's zero padding).  Direction codes (y down):
//        0:(+1,0) 1:(+1,-1) 2:(0,-1) 3:(-1,-1) 4:(-1,0) 5:(-1,+1) 6:(0,+1) 7:(+1,+1)
//  * a border is a cycle of states (pixel, dir to previous pixel a, dir to next pixel b) where b is
//    the first foreground neighbour counter-clockwise after a.  The zero neighbours strictly
//    between a and b are the ones Suzuki "examines" in that step; if code 4 (left) or 0 (right) is
//    among them the state owns the pixel's left / right crack.
//  * Suzuki starts an outer border at a foreground pixel whose left neighbour is zero and a hole
//    border at one whose right neighbour is zero, the first time the raster scan meets an
//    untraced border; equivalently the start is the raster-minimum pixel over all left/right
//    cracks of the cycle (left wins a tie) and the border is "outer" iff that crack is a left one.
//  * so: every left/right crack walks its cycle and gives up as soon as it meets a crack with a
//    raster-smaller pixel; only the canonical start survives a full lap, and it then knows the
//    contour length n.  Left cracks walk the cycle backwards, right cracks forwards (both head
//    up the image first), which kills the typical non-canonical crack within a step or two.
#pragma once
#include "common.cuh"

namespace fid {

FID_HD int dir_dx(int k) { return (int)((0x901Au >> (2 * k)) & 3u) - 1; }
FID_HD int dir_dy(int k) { return (int)((0xA901u >> (2 * k)) & 3u) - 1; }

FID_HD int rotr8(int m, int s) {
    s &= 7;
    return ((m >> s) | (m << (8 - s))) & 0xFF;
}
// first set code searching a+1, a+2, ..., a+8 (counter-clockwise); m != 0
FID_HD int next_ccw(int m, int a) {
    int t = rotr8(m, a + 1);
    return (a + 1 + fid_ctz((uint32_t)t)) & 7;
}
// first set code searching b-1, b-2, ..., b-8 (clockwise); m != 0
FID_HD int prev_cw(int m, int b) {
    int t = rotr8(m, b);
    return (b + 31 - fid_clz((uint32_t)t)) & 7;
}

enum { WALK_ABORT = 0, WALK_CANONICAL = 1, WALK_TOO_LONG = 2 };

// ---- walking representation: halo tiles + step tables -----------------------------------------------
// For walking, every plane is re-tiled into 30x30-pixel tiles stored with a 1-pixel halo as 32 words
// of 32 bits (128 bytes, one cache line): word r of tile (ty,tx) holds image row 30*ty-1+r, bit i
// holds image column 30*tx-1+i, background outside the image.  The 3x3 neighbourhood of any pixel
// then lies in ONE tile -- three loads from the line the walker already holds, no edge cases -- and
// the nine bits index a 4 KB table that returns the next direction and the examined-crack flags.
#define FID_HALO_T 30
FID_HD int div30(int v) { return (int)(((unsigned)v * 34953u) >> 20); }  // exact for 0 <= v < 2^15
FID_HD int halo_tiles_x(int W) { return (W + FID_HALO_T - 1) / FID_HALO_T; }
FID_HD size_t halo_plane_words(int W, int H) { return (size_t)halo_tiles_x(W) * ((H + FID_HALO_T - 1) / FID_HALO_T) * 32; }

struct HaloView {
    const uint32_t* base;
    int tiles_per_row;
    // 9 neighbourhood bits: bits 0-2 row y-1 (x-1,x,x+1), bits 3-5 row y, bits 6-8 row y+1
    FID_HD uint32_t idx9(int x, int y) const {
        const int qx = div30(x), qy = div30(y);
        const int i = x - FID_HALO_T * qx, r = y - FID_HALO_T * qy;
        const uint32_t* t = base + ((size_t)qy * tiles_per_row + qx) * 32 + r;
        return ((t[0] >> i) & 7u) | (((t[1] >> i) & 7u) << 3) | (((t[2] >> i) & 7u) << 6);
    }
};

FID_HD int mask_from_idx9(uint32_t v) {
    const uint32_t u = v & 7u, m = (v >> 3) & 7u, d = (v >> 6) & 7u;
    return (int)(((m >> 2) & 1u) | (((u >> 2) & 1u) << 1) | (((u >> 1) & 1u) << 2) | ((u & 1u) << 3) | ((m & 1u) << 4) | ((d & 1u) << 5) | (((d >> 1) & 1u) << 6) |
                 (((d >> 2) & 1u) << 7));
}

// Step tables, 512 neighbourhoods x 8 incoming directions, one 32-bit word each:
//   prev[idx9*8 + b] : a = first foreground neighbour clockwise from b      (backwards step)
//   next[idx9*8 + a] : b = first foreground neighbour counter-clockwise from a (forwards step)
// bits 0-2 = the direction found, bit 3 = left crack examined, bit 4 = right crack examined,
// bits 5.. = the move in that direction on a packed pixel (y << 16 | x): (dy << 16) + dx + 65537.
#define FID_LUT_SIZE 4096
FID_HD uint32_t pack_move(int dir) { return (uint32_t)(dir_dy(dir) * 65536 + dir_dx(dir) + 65537); }
inline void build_step_tables(uint32_t* prev, uint32_t* next) {
    for (int v = 0; v < 512; v++) {
        const int m = mask_from_idx9((uint32_t)v);
        for (int dir = 0; dir < 8; dir++) {
            uint32_t ep = 0, en = 0;
            if (m != 0) {
                const int a = prev_cw(m, dir);  // backwards: arrive with dir-to-next = dir
                int d = (dir - a - 1) & 7;
                ep = (uint32_t)(a | ((((4 - a - 1) & 7) < d) ? 8 : 0) | ((((0 - a - 1) & 7) < d) ? 16 : 0)) | (pack_move(a) << 5);
                const int b = next_ccw(m, dir);  // forwards: arrive with dir-to-previous = dir
                d = (b - dir - 1) & 7;
                en = (uint32_t)(b | ((((4 - dir - 1) & 7) < d) ? 8 : 0) | ((((0 - dir - 1) & 7) < d) ? 16 : 0)) | (pack_move(b) << 5);
            }
            prev[v * 8 + dir] = ep;
            next[v * 8 + dir] = en;
        }
    }
}

struct WalkCtx {
    HaloView plane;
    const uint32_t* lut_prev;
    const uint32_t* lut_next;
};

FID_HD uint32_t lut_load(const uint32_t* p) {
#if defined(__CUDA_ARCH__)
    return __ldg(p);
#else
    return *p;
#endif
}

// Walk the border owning the left (is_right=0) or right (is_right=1) crack of foreground pixel
// (x0,y0) once around.  WALK_CANONICAL with the contour point count n if (x0,y0) is the Suzuki start
// pixel of that border (outer border for a left crack, hole border for a right one); WALK_ABORT as
// soon as a crack with a raster-smaller pixel proves it is not.
//
// Direction matters for speed, not for the result: a left crack lies on a left-facing piece of
// border, where walking BACKWARDS (clockwise search) heads up the image; a right crack lies on a
// right-facing piece, where walking FORWARDS (counter-clockwise search) heads up.  Heading up
// means the very next cracks are raster-smaller, so a non-canonical start usually dies within a few
// steps (1080p marker scenes: 12-21 steps per start on average instead of 115 when every start walks
// backwards).
//
// The walk is resumable (WalkState + step budget) so that the GPU can run it in rounds of growing
// budget: a warp then only ever holds walks of similar length (kernels_contour.cuh).
enum { WALK_CONTINUE = 3 };
struct WalkState {
    int x, y;  // current pixel
    int dir;   // backwards walk: direction to the previous pixel; forwards: direction to the next pixel
    int n;     // steps taken
    int a0, b0;
};

// Returns WALK_ABORT (isolated pixel / tie lost) or WALK_CONTINUE with the state initialised.
FID_HD int walk_init(const WalkCtx& c, int x0, int y0, int is_right, WalkState* st) {
    const uint32_t v = c.plane.idx9(x0, y0);
    if ((v & ~0x10u) == 0u) return WALK_ABORT;  // isolated pixel: 1-point contour, never long enough to matter
    const int crack = is_right ? 0 : 4;
    const int a0 = lut_load(c.lut_prev + v * 8 + crack) & 7;
    const int b0 = lut_load(c.lut_next + v * 8 + crack) & 7;
    if (is_right) {  // the same state also owns the left crack -> the left-crack walker wins the tie
        const int d = (b0 - a0 - 1) & 7;
        if (((4 - a0 - 1) & 7) < d) return WALK_ABORT;
    }
    st->x = x0;
    st->y = y0;
    st->n = 0;
    st->a0 = a0;
    st->b0 = b0;
    st->dir = is_right ? b0 : a0;
    return WALK_CONTINUE;
}

// Advance by at most `budget` steps.  Returns WALK_CANONICAL (st->n = contour length), WALK_ABORT,
// WALK_TOO_LONG (more than max_len steps) or WALK_CONTINUE (budget exhausted, state updated).
struct NoVisit {
    FID_HD void operator()(int, int, bool, bool) const {}
};

// `visit(x, y, exL, exR)` is called for every state that owns a left/right crack whose pixel is raster
// larger than the start (i.e. a crack this walk has just proven non-canonical).
template <bool IS_RIGHT, class Visit = NoVisit>
FID_HD int walk_resume_dir(const WalkCtx& c, int x0, int y0, int max_len, int budget, WalkState* st, const Visit& visit = Visit()) {
    int x = st->x, y = st->y, n = st->n, dir = st->dir;
    const int ref = IS_RIGHT ? st->a0 : st->b0;  // closing condition: arrive at the start with this direction
    const uint32_t* lut = IS_RIGHT ? c.lut_next : c.lut_prev;
    const int stop_at = n + budget;
    int result = WALK_CONTINUE;
    while (n < stop_at) {
        x += dir_dx(dir);
        y += dir_dy(dir);
        n++;
        const int back = (dir + 4) & 7;
        if (x == x0 && y == y0 && back == ref) {
            result = WALK_CANONICAL;
            break;
        }
        if (n > max_len) {
            result = WALK_TOO_LONG;
            break;
        }
        const int e = lut_load(lut + c.plane.idx9(x, y) * 8 + back);
        dir = e & 7;
        if (e & 0x18) {
            if (y < y0 || (y == y0 && x < x0) || (IS_RIGHT && (e & 8) && y == y0 && x == x0)) {
                result = WALK_ABORT;
                break;
            }
            visit(x, y, (e & 8) != 0, (e & 16) != 0);
        }
    }
    st->x = x;
    st->y = y;
    st->n = n;
    st->dir = dir;
    return result;
}

// ---- bidirectional walk -------------------------------------------------------------------------------
// A start that survives the first few steps in its "uphill" direction is typically a local peak of a
// ragged border: the raster-smaller crack that disproves it may be a few steps away in EITHER
// direction, and in the wrong direction it is a whole lap away.  So from the second round on a walk
// runs a forward and a backward walker in lock step (two independent dependency chains per thread)
// and gives up as soon as either meets a raster-smaller crack: 2*min(d_fwd, d_bwd) steps instead of
// d_chosen.  The canonical start is recognised when the two walkers meet (same cycle state); the sum
// of their step counts is then the contour length.
struct WalkState2 {
    int xf, yf, df;  // forward walker: pixel, direction to the next pixel
    int xb, yb, db;  // backward walker: pixel, direction to the previous pixel
    int n;           // steps taken by both walkers together
    int nf;          // steps taken by the forward walker
};

// Continue a one-directional WalkState (walk_init / walk_resume_dir) as a bidirectional one.
template <bool IS_RIGHT>
FID_HD void walk_split(int x0, int y0, const WalkState& st, WalkState2* s2) {
    if (IS_RIGHT) {  // the forward walker has moved, the backward one still sits on the start state
        s2->xf = st.x; s2->yf = st.y; s2->df = st.dir;
        s2->xb = x0; s2->yb = y0; s2->db = st.a0;
        s2->nf = st.n;
    } else {
        s2->xb = st.x; s2->yb = st.y; s2->db = st.dir;
        s2->xf = x0; s2->yf = y0; s2->df = st.b0;
        s2->nf = 0;
    }
    s2->n = st.n;
}

// Advance both walkers by at most `budget` steps in total (budget even).  Same results as
// walk_resume_dir.
template <bool IS_RIGHT>
FID_HD int walk_resume_bidir(const WalkCtx& c, int x0, int y0, int max_len, int budget, WalkState2* st) {
    int xf = st->xf, yf = st->yf, df = st->df, xb = st->xb, yb = st->yb, db = st->db, n = st->n, nf = st->nf;
    const int stop_at = n + budget;
    int result = WALK_CONTINUE;
    while (n < stop_at) {
        // forward step
        xf += dir_dx(df);
        yf += dir_dy(df);
        n++;
        nf++;
        const int back_f = (df + 4) & 7;
        if (xf == xb && yf == yb && back_f == db) {
            result = WALK_CANONICAL;
            break;
        }
        if (n > max_len) {
            result = WALK_TOO_LONG;
            break;
        }
        // backward step (independent of the forward one: the two table look-ups overlap)
        const int xb1 = xb + dir_dx(db), yb1 = yb + dir_dy(db);
        const int back_b = (db + 4) & 7;
        const int ef = lut_load(c.lut_next + c.plane.idx9(xf, yf) * 8 + back_f);
        const int eb = lut_load(c.lut_prev + c.plane.idx9(xb1, yb1) * 8 + back_b);
        df = ef & 7;
        if ((ef & 0x18) && (yf < y0 || (yf == y0 && xf < x0) || (IS_RIGHT && (ef & 8) && yf == y0 && xf == x0))) {
            result = WALK_ABORT;
            break;
        }
        xb = xb1;
        yb = yb1;
        n++;
        if (xb == xf && yb == yf && back_b == df) {
            result = WALK_CANONICAL;
            break;
        }
        if (n > max_len) {
            result = WALK_TOO_LONG;
            break;
        }
        db = eb & 7;
        if ((eb & 0x18) && (yb < y0 || (yb == y0 && xb < x0) || (IS_RIGHT && (eb & 8) && yb == y0 && xb == x0))) {
            result = WALK_ABORT;
            break;
        }
    }
    st->xf = xf; st->yf = yf; st->df = df;
    st->xb = xb; st->yb = yb; st->db = db;
    st->n = n;
    st->nf = nf;
    return result;
}

// ---- hot-loop versions ----------------------------------------------------------------------------------
// Same walks on packed pixels (y << 16 | x: raster order is unsigned integer order) with the per-step max_len
// test hoisted out of the loop.  The lanes of a warp sit on unrelated borders, so every global load of a step is
// a 128-byte transaction of its own per active lane; the loops keep those few:
//  * a walker keeps the three tile words around its pixel in registers (TileWin).  A step moves one pixel: a
//    horizontal move loads nothing, a vertical or diagonal one loads one word, and only a move out of the
//    30 x 30 tile loads three (from the neighbouring tile, whose halo again holds the whole neighbourhood);
//  * the loops read bits 0-4 of a step-table entry (direction, crack flags) through step_load() and derive the
//    move from the direction, so that the kernels can walk on byte-per-entry copies of the tables in shared
//    memory (StepTabs<uint8_t>) while the WalkCtx overloads below read the 32-bit tables.
// What this buys on the H100 is in DESIGN.md section 4 ("What a walk step costs").
// Results are identical to walk_resume_dir / walk_resume_bidir (tests/test_hostsim_contours.py,
// tests/test_hostsim_walk_window.py).
template <class E>
struct StepTabs {
    const E* prev;
    const E* next;
};
FID_HD uint32_t step_load(const uint32_t* p) { return lut_load(p) & 31u; }
FID_HD uint32_t step_load(const uint8_t* p) { return *p; }
inline void build_step_bytes(uint8_t* prev, uint8_t* next) {
    uint32_t p[FID_LUT_SIZE], n[FID_LUT_SIZE];
    build_step_tables(p, n);
    for (int k = 0; k < FID_LUT_SIZE; k++) {
        prev[k] = (uint8_t)(p[k] & 31u);
        next[k] = (uint8_t)(n[k] & 31u);
    }
}

struct TileWin {
    uint32_t o;           // word offset of the walker's tile in the plane
    int r, i;             // the pixel is bit i + 1 of word r + 1 of that tile, 0 <= r, i < FID_HALO_T
    uint32_t w0, w1, w2;  // words r, r + 1, r + 2
    FID_HD void load(const uint32_t* plane) {
        const uint32_t* t = plane + o + r;
        w0 = t[0];
        w1 = t[1];
        w2 = t[2];
    }
    FID_HD void enter(const uint32_t* plane, uint32_t tiles_per_row, uint32_t xy) {
        const uint32_t x = xy & 0xFFFFu, y = xy >> 16;
        const uint32_t qx = (x * 34953u) >> 20, qy = (y * 34953u) >> 20;
        o = (qy * tiles_per_row + qx) * 32u;
        r = (int)(y - FID_HALO_T * qy);
        i = (int)(x - FID_HALO_T * qx);
        load(plane);
    }
    // from a tile index and the word / bit of the pixel inside the tile (1 .. FID_HALO_T: what a start record holds)
    FID_HD void enter_tile(const uint32_t* plane, uint32_t tile, uint32_t row, uint32_t col) {
        o = tile * 32u;
        r = (int)row - 1;
        i = (int)col - 1;
        load(plane);
    }
    FID_HD uint32_t idx9() const { return ((w0 >> i) & 7u) | (((w1 >> i) & 7u) << 3) | (((w2 >> i) & 7u) << 6); }
    // Move by (dx, dy), each in -1 .. 1, to a pixel inside the image.
    FID_HD void step(const uint32_t* plane, uint32_t tiles_per_row, int dx, int dy) {
        i += dx;
        r += dy;
        if ((unsigned)i >= (unsigned)FID_HALO_T || (unsigned)r >= (unsigned)FID_HALO_T) {
            if (i < 0) {
                i = FID_HALO_T - 1;
                o -= 32u;
            } else if (i >= FID_HALO_T) {
                i = 0;
                o += 32u;
            }
            if (r < 0) {
                r = FID_HALO_T - 1;
                o -= tiles_per_row * 32u;
            } else if (r >= FID_HALO_T) {
                r = 0;
                o += tiles_per_row * 32u;
            }
            load(plane);
        } else if (dy != 0) {
            const uint32_t nw = plane[o + (uint32_t)(r + 1 + dy)];
            const uint32_t mid = dy > 0 ? w2 : w0;
            w0 = dy > 0 ? w1 : nw;
            w2 = dy > 0 ? nw : w1;
            w1 = mid;
        }
    }
};
FID_HD uint32_t move_of(int dx, int dy) { return (uint32_t)(dy * 65536 + dx); }

// walk_init on a neighbourhood already read (v = idx9 of the start pixel).
template <class E>
FID_HD int walk_init_at(uint32_t v, const StepTabs<E>& tabs, int x0, int y0, int is_right, WalkState* st) {
    if ((v & ~0x10u) == 0u) return WALK_ABORT;
    const int crack = is_right ? 0 : 4;
    const int a0 = (int)(step_load(tabs.prev + v * 8 + crack) & 7u);
    const int b0 = (int)(step_load(tabs.next + v * 8 + crack) & 7u);
    if (is_right) {
        const int d = (b0 - a0 - 1) & 7;
        if (((4 - a0 - 1) & 7) < d) return WALK_ABORT;
    }
    st->x = x0;
    st->y = y0;
    st->n = 0;
    st->a0 = a0;
    st->b0 = b0;
    st->dir = is_right ? b0 : a0;
    return WALK_CONTINUE;
}

// One-directional walk of at most `budget` steps (round 0).  `w` sits on the walker's pixel (st->x, st->y) and
// follows it; lut = the table of the walk's direction (IS_RIGHT ? next : prev).
template <bool IS_RIGHT, class E>
FID_HD int walk_uni_fast(const uint32_t* plane, uint32_t tpr, const E* lut, TileWin& w, int x0, int y0, int max_len, int budget, WalkState* st) {
    const uint32_t xy0 = (uint32_t)x0 | ((uint32_t)y0 << 16);
    const uint32_t ref = (uint32_t)(IS_RIGHT ? st->a0 : st->b0);
    uint32_t xy = (uint32_t)st->x | ((uint32_t)st->y << 16);
    uint32_t d = (uint32_t)st->dir;
    int result = WALK_CONTINUE, k = 0;
    for (; k < budget; k++) {
        const int dx = dir_dx((int)d), dy = dir_dy((int)d);
        xy += move_of(dx, dy);
        const uint32_t back = d ^ 4u;
        if (xy == xy0 && back == ref) {
            result = WALK_CANONICAL;
            k++;
            break;
        }
        w.step(plane, tpr, dx, dy);
        const uint32_t e = step_load(lut + w.idx9() * 8u + back);
        d = e & 7u;
        if ((e & 0x18u) && (xy < xy0 || (IS_RIGHT && (e & 8u) && xy == xy0))) {
            result = WALK_ABORT;
            k++;
            break;
        }
    }
    st->x = (int)(xy & 0xFFFFu);
    st->y = (int)(xy >> 16);
    st->dir = (int)d;
    st->n += k;
    if (st->n > max_len && result != WALK_ABORT) result = WALK_TOO_LONG;
    return result;
}
template <bool IS_RIGHT>
FID_HD int walk_uni_fast(const WalkCtx& c, int x0, int y0, int max_len, int budget, WalkState* st) {
    const uint32_t tpr = (uint32_t)c.plane.tiles_per_row;
    TileWin w;
    w.enter(c.plane.base, tpr, (uint32_t)st->x | ((uint32_t)st->y << 16));
    return walk_uni_fast<IS_RIGHT>(c.plane.base, tpr, IS_RIGHT ? c.lut_next : c.lut_prev, w, x0, y0, max_len, budget, st);
}

// Bidirectional walk of at most `budget` steps (budget/2 lock-step iterations).  wf / wb sit on the forward and
// the backward walker's pixel and follow them while the walk continues.
template <bool IS_RIGHT, class E>
FID_HD int walk_bidir_fast(const uint32_t* plane, uint32_t tpr, const StepTabs<E>& tabs, TileWin& wf, TileWin& wb, int x0, int y0, int max_len, int budget,
                           WalkState2* st) {
    const uint32_t xy0 = (uint32_t)x0 | ((uint32_t)y0 << 16);
    uint32_t xyf = (uint32_t)st->xf | ((uint32_t)st->yf << 16), xyb = (uint32_t)st->xb | ((uint32_t)st->yb << 16);
    uint32_t df = (uint32_t)st->df, db = (uint32_t)st->db;
    const int iters = (budget + 1) >> 1;
    int result = WALK_CONTINUE, it = 0, half = 0;
    for (; it < iters; it++) {
        // both moves and both table look-ups first (two independent chains), then the tests in walk order
        const int dxf = dir_dx((int)df), dyf = dir_dy((int)df), dxb = dir_dx((int)db), dyb = dir_dy((int)db);
        const uint32_t xyf1 = xyf + move_of(dxf, dyf), xyb1 = xyb + move_of(dxb, dyb);
        const uint32_t back_f = df ^ 4u, back_b = db ^ 4u;
        wf.step(plane, tpr, dxf, dyf);
        wb.step(plane, tpr, dxb, dyb);
        const uint32_t ef1 = step_load(tabs.next + wf.idx9() * 8u + back_f);
        const uint32_t eb1 = step_load(tabs.prev + wb.idx9() * 8u + back_b);
        xyf = xyf1;
        if (xyf1 == xyb && back_f == db) {  // the forward walker arrived on the backward walker's state
            result = WALK_CANONICAL;
            half = 1;
            break;
        }
        df = ef1 & 7u;
        if ((ef1 & 0x18u) && (xyf1 < xy0 || (IS_RIGHT && (ef1 & 8u) && xyf1 == xy0))) {
            result = WALK_ABORT;
            half = 1;
            break;
        }
        xyb = xyb1;
        if (xyb1 == xyf1 && back_b == df) {  // the backward walker arrived on the forward walker's new state
            result = WALK_CANONICAL;
            half = 2;
            break;
        }
        db = eb1 & 7u;
        if ((eb1 & 0x18u) && (xyb1 < xy0 || (IS_RIGHT && (eb1 & 8u) && xyb1 == xy0))) {
            result = WALK_ABORT;
            half = 2;
            break;
        }
    }
    st->xf = (int)(xyf & 0xFFFFu);
    st->yf = (int)(xyf >> 16);
    st->df = (int)df;
    st->xb = (int)(xyb & 0xFFFFu);
    st->yb = (int)(xyb >> 16);
    st->db = (int)db;
    st->n += 2 * it + half;
    st->nf += it + (half ? 1 : 0);
    if (st->n > max_len && result != WALK_ABORT) result = WALK_TOO_LONG;
    return result;
}
template <bool IS_RIGHT>
FID_HD int walk_bidir_fast(const WalkCtx& c, int x0, int y0, int max_len, int budget, WalkState2* st) {
    const uint32_t tpr = (uint32_t)c.plane.tiles_per_row;
    TileWin wf, wb;
    wf.enter(c.plane.base, tpr, (uint32_t)st->xf | ((uint32_t)st->yf << 16));
    wb.enter(c.plane.base, tpr, (uint32_t)st->xb | ((uint32_t)st->yb << 16));
    return walk_bidir_fast<IS_RIGHT>(c.plane.base, tpr, StepTabs<uint32_t>{c.lut_prev, c.lut_next}, wf, wb, x0, y0, max_len, budget, st);
}

FID_HD int walk_resume(const WalkCtx& c, int x0, int y0, int is_right, int max_len, int budget, WalkState* st) {
    return is_right ? walk_resume_dir<true>(c, x0, y0, max_len, budget, st) : walk_resume_dir<false>(c, x0, y0, max_len, budget, st);
}

// One-shot walk (CPU harness, small inputs).  *steps_out (optional) returns the steps taken.
FID_HD int walk_start(const WalkCtx& c, int x0, int y0, int is_right, int max_len, int* n_out, int* steps_out = nullptr) {
    WalkState st;
    if (steps_out) *steps_out = 0;
    if (walk_init(c, x0, y0, is_right, &st) == WALK_ABORT) return WALK_ABORT;
    const int r = walk_resume(c, x0, y0, is_right, max_len, 0x3fffffff, &st);
    if (steps_out) *steps_out = st.n;
    if (r == WALK_CANONICAL) *n_out = st.n;
    return r;
}

// Emit the n contour points in OpenCV order (start pixel first, then Suzuki's direction).  Points are
// written four at a time (16-byte stores); `out` must be 16-byte aligned and have room for n rounded
// up to a multiple of 4.
FID_HD void trace_forward(const WalkCtx& c, int x0, int y0, int is_right, int n, Pt16* out) {
    const uint32_t v = c.plane.idx9(x0, y0);
    int x = x0, y = y0;
    if ((v & ~0x10u) == 0u) {
        out[0].x = (int16_t)x;
        out[0].y = (int16_t)y;
        return;
    }
    int a = lut_load(c.lut_prev + v * 8 + (is_right ? 0 : 4)) & 7;
    uint32_t cur = v;
    uint32_t buf[4];
    uint32_t* out32 = reinterpret_cast<uint32_t*>(out);
    for (int i = 0; i < n; i++) {
        buf[i & 3] = (uint32_t)(uint16_t)x | ((uint32_t)(uint16_t)y << 16);
        if ((i & 3) == 3) {
#if defined(__CUDA_ARCH__)
            *reinterpret_cast<uint4*>(out32 + i - 3) = make_uint4(buf[0], buf[1], buf[2], buf[3]);
#else
            for (int k = 0; k < 4; k++) out32[i - 3 + k] = buf[k];
#endif
        }
        const int b = lut_load(c.lut_next + cur * 8 + a) & 7;
        x += dir_dx(b);
        y += dir_dy(b);
        a = (b + 4) & 7;
        cur = c.plane.idx9(x, y);
    }
    for (int k = 0; k < (n & 3); k++) out32[(n & ~3) + k] = buf[k];
}

// ---- contour emission in segments ------------------------------------------------------------------
// A contour found by the bidirectional walk (length n, the forward walker took nf of the steps) is
// written by several independent threads: the points 0 .. nf-1 forwards from the start state, the
// points n-1 .. nf backwards from it, and -- for long contours -- each half again cut at the
// checkpoints the walkers dropped every FID_CKPT_STEP steps.  A segment is (state, count, index of
// the state's own point); the order of the points is cv2.findContours' (start pixel first, Suzuki's
// direction).
#define FID_CKPT_STEP 256
#define FID_CKPT_MAX 16
struct SegRec {
    uint32_t xy;    // pixel of the state
    uint32_t meta;  // frame << 8 | scale << 1 | backward
    uint32_t dn;    // dir | count << 3: forward segment -> dir to the next pixel, backward -> dir to the previous one
    uint32_t off;   // index of the state's own point in the point buffer
};
struct WalkCkpt {
    // side 0: forward walker, side 1: backward walker; dn = dir | (steps that walker had taken) << 3
    uint32_t xy[2][FID_CKPT_MAX];
    uint32_t dn[2][FID_CKPT_MAX];
    int count[2];
};

// forward: points[off + t] = pixel after t steps, t = 0 .. count-1
// backward: points[off - t] = pixel after t steps, t = 1 .. count
// Points are written in ascending-address groups of four words that start at a multiple of four (one 16-byte
// store each; `points` is 16-byte aligned), single words before the first and after the last full group of
// the segment: a segment never writes a word that is not its own.
FID_HD void store_points4(uint32_t* p, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
#if defined(__CUDA_ARCH__)
    *reinterpret_cast<uint4*>(p) = make_uint4(a, b, c, d);
#else
    p[0] = a;
    p[1] = b;
    p[2] = c;
    p[3] = d;
#endif
}
template <class E>
FID_HD void trace_segment(const uint32_t* plane, uint32_t tpr, const StepTabs<E>& tabs, const SegRec& s, uint32_t* points) {
    const bool backward = (s.meta & 1u) != 0u;
    const E* lut = backward ? tabs.prev : tabs.next;
    const int count = (int)(s.dn >> 3);
    uint32_t xy = s.xy, d = s.dn & 7u;
    TileWin w;
    w.enter(plane, tpr, xy);
    // the walker's next point: a forward segment starts with the state's own pixel, a backward one with the first move
    auto next_point = [&]() {
        const int dx = dir_dx((int)d), dy = dir_dy((int)d);
        const uint32_t cur = xy;
        xy += move_of(dx, dy);
        w.step(plane, tpr, dx, dy);
        d = step_load(lut + w.idx9() * 8u + (d ^ 4u)) & 7u;
        return backward ? xy : cur;
    };
    int t = 0;
    if (backward) {  // words off-1, off-2, ..., off-count
        uint32_t at = s.off;  // one past the next word to write
        for (; t < count && (at & 3u); t++) points[--at] = next_point();
        for (; t + 4 <= count; t += 4) {
            const uint32_t p3 = next_point(), p2 = next_point(), p1 = next_point(), p0 = next_point();
            at -= 4;
            store_points4(points + at, p0, p1, p2, p3);
        }
        for (; t < count; t++) points[--at] = next_point();
    } else {  // words off, off+1, ..., off+count-1
        uint32_t at = s.off;
        for (; t < count && (at & 3u); t++) points[at++] = next_point();
        for (; t + 4 <= count; t += 4) {
            const uint32_t p0 = next_point(), p1 = next_point(), p2 = next_point(), p3 = next_point();
            store_points4(points + at, p0, p1, p2, p3);
            at += 4;
        }
        for (; t < count; t++) points[at++] = next_point();
    }
}
FID_HD void trace_segment(const WalkCtx& c, const SegRec& s, uint32_t* points) {
    trace_segment(c.plane.base, (uint32_t)c.plane.tiles_per_row, StepTabs<uint32_t>{c.lut_prev, c.lut_next}, s, points);
}

// Number of segments of a contour, and the segments themselves (sink(k, SegRec) for k = 0 .. count-1).
FID_HD int segment_count(const WalkCkpt* ck) { return 2 + (ck ? ck->count[0] + ck->count[1] : 0); }
template <class Sink>
FID_HD void make_segments(const WalkCtx& c, int x0, int y0, int is_right, int n, int nf, const WalkCkpt* ck, uint32_t meta_fs, uint32_t chain_off, const Sink& sink) {
    const uint32_t v = c.plane.idx9(x0, y0);
    const int crack = is_right ? 0 : 4;
    const int a0 = lut_load(c.lut_prev + v * 8 + crack) & 7, b0 = lut_load(c.lut_next + v * 8 + crack) & 7;
    const uint32_t xy0 = (uint32_t)x0 | ((uint32_t)y0 << 16);
    const uint32_t meta = meta_fs & ~1u;
    int k = 0;
    {  // forward half: points 0 .. nf-1
        uint32_t xy = xy0;
        int dir = b0, at = 0;
        const int m = ck ? ck->count[0] : 0;
        for (int i = 0; i <= m; i++) {
            const int next_at = i < m ? (int)(ck->dn[0][i] >> 3) : nf;
            sink(k++, SegRec{xy, meta, (uint32_t)dir | ((uint32_t)(next_at - at) << 3), chain_off + (uint32_t)at});
            if (i < m) {
                xy = ck->xy[0][i];
                dir = (int)(ck->dn[0][i] & 7);
                at = next_at;
            }
        }
    }
    {  // backward half: points n-1 .. nf
        uint32_t xy = xy0;
        int dir = a0, at = 0;  // at = steps the backward walker had taken
        const int nb = n - nf;
        const int m = ck ? ck->count[1] : 0;
        for (int i = 0; i <= m; i++) {
            const int next_at = i < m ? (int)(ck->dn[1][i] >> 3) : nb;
            sink(k++, SegRec{xy, meta | 1u, (uint32_t)dir | ((uint32_t)(next_at - at) << 3), chain_off + (uint32_t)(n - at)});
            if (i < m) {
                xy = ck->xy[1][i];
                dir = (int)(ck->dn[1][i] & 7);
                at = next_at;
            }
        }
    }
}

// Drop checkpoints of both walkers when they have moved FID_CKPT_STEP steps since their last one.
FID_HD void walk_checkpoint(const WalkState2& st, WalkCkpt* ck, int* last_f, int* last_b, int step = FID_CKPT_STEP) {
    const int nb = st.n - st.nf;
    if (st.nf - *last_f >= step && ck->count[0] < FID_CKPT_MAX) {
        const int i = ck->count[0]++;
        ck->xy[0][i] = (uint32_t)st.xf | ((uint32_t)st.yf << 16);
        ck->dn[0][i] = (uint32_t)st.df | ((uint32_t)st.nf << 3);
        *last_f = st.nf;
    }
    if (nb - *last_b >= step && ck->count[1] < FID_CKPT_MAX) {
        const int i = ck->count[1]++;
        ck->xy[1][i] = (uint32_t)st.xb | ((uint32_t)st.yb << 16);
        ck->dn[1][i] = (uint32_t)st.db | ((uint32_t)nb << 3);
        *last_b = nb;
    }
}

// ---- start cracks of one halo-tile row -----------------------------------------------------------------
// up / mid / dn = words r-1 / r / r+1 of a tile (r = 1..30); only interior bits 1..30 are reported.  Every
// left/right crack is a potential Suzuki start; the ones that a walk would discard within its first
// step are removed here with bit operations (all rules are exact -- they only drop cracks whose
// walk provably aborts, so the set of canonical starts is unchanged):
//   L0  pixel above is foreground with a zero left neighbour        -> that crack dominates
//   L1  up, up-left zero and up-right foreground                     -> first backward step lands on
//       (x+1,y-1), whose left neighbour (x,y-1) is an examined zero: raster-smaller left crack
//   L2  up-left foreground, (x-2,y) and (x-2,y-1) zero               -> first backward step lands on
//       (x-1,y-1) which owns a left crack
// and the mirror images R0..R2 for right cracks (forward walk); I0 drops isolated pixels.
FID_HD void halo_row_starts(uint32_t up, uint32_t mid, uint32_t dn, uint32_t* L, uint32_t* R) {
    const uint32_t interior = 0x7FFFFFFEu;
    const uint32_t up_l = up << 1, up_r = up >> 1, mid_l = mid << 1, mid_r = mid >> 1;
    // I0: an isolated pixel is a 1-point contour (walk_init gives up on it)
    const uint32_t lone = mid & ~(up | up_l | up_r | mid_l | mid_r | dn | (dn << 1) | (dn >> 1));
    uint32_t l = mid & ~mid_l & ~(up & ~up_l) & ~lone;
    l &= ~(~up & ~up_l & up_r);
    l &= ~(up_l & ~(mid << 2) & ~(up << 2) & 0xFFFFFFFCu);
    uint32_t r = mid & ~mid_r & ~(up & ~up_r) & ~lone;
    r &= ~(~up & ~up_r & up_l);
    r &= ~(up_r & ~(mid >> 2) & ~(up >> 2) & 0x3FFFFFFFu);
    *L = l & interior;
    *R = r & interior;
}

// Second, optional pruning stage (start_prune_table.h, tools/gen_prune_table.py): the 3 x 5 neighbourhood of a surviving start
// indexes a table of the patterns for which the start's walk provably aborts within 3 steps whatever lies outside the
// neighbourhood (exhaustively enumerated with the walk code itself).  tab = kStartPruneTable laid out [2][FID_START_PRUNE_WORDS].
// Columns 1 and 30 of a tile are left alone: their neighbourhood reaches beyond the halo.
FID_HD void halo_prune_starts(uint32_t up, uint32_t mid, uint32_t dn, uint32_t* L, uint32_t* R, const uint32_t* tab) {
    for (int side = 0; side < 2; side++) {
        uint32_t* S = side ? R : L;
        uint32_t todo = *S & 0x3FFFFFFCu;  // columns 2..29
        const uint32_t* t = tab + side * 1024;
        while (todo) {
            const int i = fid_ctz(todo);
            todo &= todo - 1;
            const uint32_t pat = ((up >> (i - 2)) & 31u) | (((mid >> (i - 2)) & 31u) << 5) | (((dn >> (i - 2)) & 31u) << 10);
            if ((lut_load(t + (pat >> 5)) >> (pat & 31u)) & 1u) *S &= ~(1u << i);
        }
    }
}

}  // namespace fid
