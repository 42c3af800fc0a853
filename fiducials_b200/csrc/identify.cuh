// Marker identification for one quad candidate: perspective removal (nearest warp), Otsu, cell
// votes, border check and first-match dictionary search -- cv::aruco::_identifyOneCandidate /
// _extractBits / Dictionary::identify (OpenCV 4.13 semantics, SURVEY.md A.6-A.7), executed by the
// reference at aruco_detect/src/aruco_detect.cpp:350.
//
// Written SPMD over a "lane group" (a CUDA warp in the kernel, a single lane in tests/hostsim):
// pixels / cells / dictionary entries are strided over lanes, integer reductions go through the
// Lanes object.  All floating point that decides a pixel or a bit is double and evaluated in the
// same association order as OpenCV (no FMA: the library is built with --fmad=false).
#pragma once
#include "common.cuh"
#include "quad_group.cuh"

namespace fid {

struct SerialLanes {
    FID_HD int lane() const { return 0; }
    FID_HD int count() const { return 1; }
    FID_HD void sync() const {}
    FID_HD long long sum(long long v) const { return v; }
    FID_HD int min_i(int v) const { return v; }
    FID_HD unsigned long long or_u64(unsigned long long v) const { return v; }
    FID_HD void hist_add(int* h, int bin) const { h[bin]++; }
    FID_HD uint32_t ballot(bool p) const { return p ? 1u : 0u; }
    FID_HD int shfl_i(int v, int) const { return v; }
    FID_HD int atomic_add(int* p, int v) const {
        const int old = *p;
        *p += v;
        return old;
    }
};

// getPerspectiveTransform(src quad -> dst square) : 8x8 LU with partial pivoting, double.
FID_HD bool perspective_transform(const QuadF& q, double size_minus_1, double M[9]) {
    double A[8][8], B[8];
    const double dx[4] = {0.0, size_minus_1, size_minus_1, 0.0};
    const double dy[4] = {0.0, 0.0, size_minus_1, size_minus_1};
    for (int i = 0; i < 4; i++) {
        const double sx = q.x[i], sy = q.y[i];
        A[i][0] = A[i + 4][3] = sx;
        A[i][1] = A[i + 4][4] = sy;
        A[i][2] = A[i + 4][5] = 1.0;
        A[i][3] = A[i][4] = A[i][5] = A[i + 4][0] = A[i + 4][1] = A[i + 4][2] = 0.0;
        A[i][6] = -sx * dx[i];
        A[i][7] = -sy * dx[i];
        A[i + 4][6] = -sx * dy[i];
        A[i + 4][7] = -sy * dy[i];
        B[i] = dx[i];
        B[i + 4] = dy[i];
    }
    for (int i = 0; i < 8; i++) {
        int k = i;
        for (int j = i + 1; j < 8; j++)
            if (fabs(A[j][i]) > fabs(A[k][i])) k = j;
        if (fabs(A[k][i]) < 2.220446049250313e-16 * 100) return false;
        if (k != i) {
            for (int j = i; j < 8; j++) {
                const double t = A[i][j];
                A[i][j] = A[k][j];
                A[k][j] = t;
            }
            const double t = B[i];
            B[i] = B[k];
            B[k] = t;
        }
        const double d = -1.0 / A[i][i];
        for (int j = i + 1; j < 8; j++) {
            const double alpha = A[j][i] * d;
            for (int c = i + 1; c < 8; c++) A[j][c] += alpha * A[i][c];
            B[j] += alpha * B[i];
        }
    }
    for (int i = 7; i >= 0; i--) {
        double s = B[i];
        for (int c = i + 1; c < 8; c++) s -= A[i][c] * B[c];
        B[i] = s / A[i][i];
    }
    for (int i = 0; i < 8; i++) M[i] = B[i];
    M[8] = 1.0;
    return true;
}

// cv::invert of a 3x3 double matrix (cofactors times 1/det).
FID_HD bool invert3x3(const double S[9], double T[9]) {
    double d = S[0] * (S[4] * S[8] - S[5] * S[7]) - S[1] * (S[3] * S[8] - S[5] * S[6]) + S[2] * (S[3] * S[7] - S[4] * S[6]);
    if (d == 0.0) return false;
    d = 1.0 / d;
    T[0] = (S[4] * S[8] - S[5] * S[7]) * d;
    T[1] = (S[2] * S[7] - S[1] * S[8]) * d;
    T[2] = (S[1] * S[5] - S[2] * S[4]) * d;
    T[3] = (S[5] * S[6] - S[3] * S[8]) * d;
    T[4] = (S[0] * S[8] - S[2] * S[6]) * d;
    T[5] = (S[2] * S[3] - S[0] * S[5]) * d;
    T[6] = (S[3] * S[7] - S[4] * S[6]) * d;
    T[7] = (S[1] * S[6] - S[0] * S[7]) * d;
    T[8] = (S[0] * S[4] - S[1] * S[3]) * d;
    return true;
}

FID_HD int round_half_even_to_int(double v) {
#if defined(__CUDA_ARCH__)
    return __double2int_rn(v);
#else
    return (int)nearbyint(v);  // default rounding mode = to nearest even
#endif
}

// warpPerspective(INTER_NEAREST, BORDER_CONSTANT 0) sample for destination pixel (x,y).
template <class Img>
FID_HD int warp_nearest_sample(const Img& gray, int W, int H, const double Mi[9], int x, int y) {
    const double X0 = Mi[1] * y + Mi[2];
    const double Y0 = Mi[4] * y + Mi[5];
    const double W0 = Mi[7] * y + Mi[8];
    double w = W0 + Mi[6] * x;
    w = w != 0.0 ? 1.0 / w : 0.0;
    double fx = (X0 + Mi[0] * x) * w;
    double fy = (Y0 + Mi[3] * x) * w;
    fx = fx < -2147483648.0 ? -2147483648.0 : (fx > 2147483647.0 ? 2147483647.0 : fx);
    fy = fy < -2147483648.0 ? -2147483648.0 : (fy > 2147483647.0 ? 2147483647.0 : fy);
    const int sx = round_half_even_to_int(fx), sy = round_half_even_to_int(fy);
    if ((unsigned)sx < (unsigned)W && (unsigned)sy < (unsigned)H) return gray.at(sx, sy);
    return 0;
}

// Otsu threshold over a 256-bin histogram of `total` samples (first maximum wins).
FID_HD int otsu_threshold(const int* h, int total) {
    double mu = 0.0;
    const double scale = 1.0 / (double)total;
    for (int i = 0; i < 256; i++) mu += i * (double)h[i];
    mu *= scale;
    double mu1 = 0.0, q1 = 0.0, max_sigma = 0.0;
    int max_val = 0;
    for (int i = 0; i < 256; i++) {
        const double p_i = h[i] * scale;
        mu1 *= q1;
        q1 += p_i;
        const double q2 = 1.0 - q1;
        const double lo = q1 < q2 ? q1 : q2, hi = q1 < q2 ? q2 : q1;
        if (lo < 1.1920928955078125e-07 || hi > 1.0 - 1.1920928955078125e-07) continue;
        mu1 = (mu1 + i * p_i) / q1;
        const double mu2 = (mu - q1 * mu1) / q2;
        const double sigma = q1 * q2 * (mu1 - mu2) * (mu1 - mu2);
        if (sigma > max_sigma) {
            max_sigma = sigma;
            max_val = i;
        }
    }
    return max_val;
}

struct IdentifyResult {
    int id;         // -1 = rejected
    int rotation;   // number of corner rotations to apply
    bool inverted;  // detectInvertedMarker: the cells were read inverted (a white marker on a dark surround)
};

// The cell bits of a quad (_extractBits): cell c = y*cells + x is bit c of lo for c < 64, bit c-64 of hi otherwise (7x7 markers
// have 81 cells).
struct CellBits {
    unsigned long long lo, hi;
    bool ok;  // false: the quad gives no perspective transform
    FID_HD int at(int c) const { return (int)(((c < 64 ? lo >> c : hi >> (c - 64))) & 1ull); }
};

// _extractBits: perspective removal (nearest warp), Otsu or the minOtsuStdDev rule, cell votes.  ok = false where the quad
// gives no perspective transform.  Returned by value: through an out pointer k_identify_first spilled more.
// `img` : S*S bytes of scratch, `hist`: 256 ints of scratch (zeroed by this function).
// CONF (detectMarkersWithConfidence): where ok, hist[c] holds on return cell c's count of window pixels above the threshold --
// the whole window (win^2) or none in the minOtsuStdDev rule, as the bits there.
template <bool CONF = false, class Lanes, class Img>
FID_HD CellBits extract_bits(const Lanes& L, const Img& gray, int W, int H, const QuadF& quad, const DevParams& P, uint8_t* img, int* hist) {
    CellBits out = {0ull, 0ull, false};
    const int cells = P.marker_size + 2 * P.marker_border_bits;
    const int cell = P.px_per_cell;
    const int S = cells * cell;
    const int margin = (int)(P.ignored_margin_per_cell * cell);
    double M[9], Mi[9];
    if (!perspective_transform(quad, (double)(S - 1), M)) return out;
    if (!invert3x3(M, Mi)) return out;
    for (int i = L.lane(); i < 256; i += L.count()) hist[i] = 0;
    L.sync();
    const int half = cell / 2;
    long long s1 = 0, s2 = 0;
    for (int p = L.lane(); p < S * S; p += L.count()) {
        const int y = p / S, x = p - y * S;
        const int v = warp_nearest_sample(gray, W, H, Mi, x, y);
        img[p] = (uint8_t)v;
        L.hist_add(hist, v);
        if (x >= half && x < S - half && y >= half && y < S - half) {
            s1 += v;
            s2 += v * v;
        }
    }
    s1 = L.sum(s1);
    s2 = L.sum(s2);
    L.sync();
    // meanStdDev of the inner region
    const int inner = (S - 2 * half) * (S - 2 * half);
    const double scale = 1.0 / (double)inner;
    const double mean = (double)s1 * scale;
    double var = (double)s2 * scale - mean * mean;
    var = var > 0.0 ? var : 0.0;
    const double stddev = sqrt(var);
    unsigned long long bits_lo = 0, bits_hi = 0;
    if (stddev < P.min_otsu_stddev) {
        if (mean > 127.0) bits_lo = bits_hi = ~0ull;  // all white (bits beyond cells*cells are never read)
        if constexpr (CONF) {
            const int win = cell - 2 * margin;
            L.sync();  // every lane is done with the histogram
            for (int c = L.lane(); c < cells * cells; c += L.count()) hist[c] = mean > 127.0 ? win * win : 0;
            L.sync();
        }
    } else {
        const int t = otsu_threshold(hist, S * S);
        const int win = cell - 2 * margin;
        if constexpr (CONF) L.sync();  // every lane has read the histogram
        unsigned long long mine = 0, mine_hi = 0;
        for (int c = L.lane(); c < cells * cells; c += L.count()) {
            const int cy = c / cells, cx = c - cy * cells;
            int nz = 0;
            for (int yy = 0; yy < win; yy++)
                for (int xx = 0; xx < win; xx++) nz += img[(cy * cell + margin + yy) * S + cx * cell + margin + xx] > t ? 1 : 0;
            if constexpr (CONF) hist[c] = nz;
            if (nz > (win * win) / 2) {
                if (c < 64)
                    mine |= 1ull << c;
                else
                    mine_hi |= 1ull << (c - 64);
            }
        }
        bits_lo = L.or_u64(mine);
        bits_hi = cells * cells > 64 ? L.or_u64(mine_hi) : 0ull;
        if constexpr (CONF) L.sync();
    }
    out.lo = bits_lo;
    out.hi = bits_hi;
    out.ok = true;
    return out;
}

// The inner bits as a byte list (getByteListFromBits: row-major, MSB first, last partial byte right aligned) packed into a u64 the
// way the dictionary words are.
FID_HD unsigned long long inner_code(const CellBits& b, const DevParams& P) {
    const int cells = P.marker_size + 2 * P.marker_border_bits;
    const int bb = P.marker_border_bits, ms = P.marker_size;
    unsigned long long cand = 0;
    int k = 0, cur = 0, nbits = 0, byte_i = 0;
    const int total = ms * ms;
    for (int y = 0; y < ms; y++)
        for (int x = 0; x < ms; x++) {
            cur = (cur << 1) | b.at((y + bb) * cells + x + bb);
            nbits++;
            k++;
            if (nbits == 8 || k == total) {
                cand |= (unsigned long long)cur << (8 * byte_i);
                byte_i++;
                cur = 0;
                nbits = 0;
            }
        }
    return cand;
}

// detectMarkersWithConfidence (DESIGN.md finding 17): 1 - the mean over the cells of the share of each cell's window that
// disagrees with the decoded marker -- black in the border, inside the dictionary word `word` as identify_candidate matched it
// (the rotation seen in the canonical image).  Not the extracted bits: an inner cell that error correction fixed costs its
// whole share.  cnt = extract_bits<true>'s counts.  Each cell's share is a float; their sum is exact in double (81 floats in
// [0, 1] whose exponents span less than 53 bits) and rounded once to float before the float division: independent of the order,
// so the kernels and the host agree bit for bit.  cv2's own order is not pinned; where win^2 is not a power of two the two can
// differ in the last float bit.
FID_HD float marker_confidence(const int* cnt, const DevParams& P, unsigned long long word) {
    const int bb = P.marker_border_bits, ms = P.marker_size, cells = ms + 2 * bb;
    const int margin = (int)(P.ignored_margin_per_cell * P.px_per_cell);
    const int win = P.px_per_cell - 2 * margin;
    const float area = (float)(win * win);
    const int total = ms * ms, last_byte = (total - 1) >> 3, last_bits = total & 7 ? total & 7 : 8;
    double sum = 0.0;
    for (int y = 0; y < cells; y++)
        for (int x = 0; x < cells; x++) {
            const float ratio = (float)cnt[y * cells + x] / area;
            bool one = false;
            if (y >= bb && y < cells - bb && x >= bb && x < cells - bb) {  // inner_code's packing: row-major, MSB first per byte
                const int k = (y - bb) * ms + x - bb, byte = k >> 3;
                const int nb = byte == last_byte ? last_bits : 8;
                one = (word >> (8 * byte + nb - 1 - (k & 7))) & 1ull;
            }
            sum += one ? 1.0f - ratio : ratio;
        }
    return 1.0f - (float)sum / (float)(cells * cells);
}

// `img` : S*S bytes of scratch, `hist`: 256 ints of scratch (zeroed by this function).
// dict  : n_markers x 4 rotations packed as little-endian byte strings in 64-bit words.
// CONF: on a match hist holds the cell counts marker_confidence reads, with word dict[id * 4 + rotation].
// INV (detectInvertedMarker, DESIGN.md finding 18 A): the border errors are also counted on the inverted cells, and where they are
// strictly fewer the candidate continues as a white marker -- the inverted cells go to the border limit and the dictionary search,
// and under CONF the counts become the inverted window's (win^2 - count), so that the confidence is measured against the polarity
// that was chosen.  A tie keeps the cells as read.
template <bool CONF = false, bool INV = false, class Lanes, class Img>
FID_HD IdentifyResult identify_candidate(const Lanes& L, const Img& gray, int W, int H, const QuadF& quad, const DevParams& P, const unsigned long long* dict, uint8_t* img,
                                         int* hist) {
    IdentifyResult res = {-1, 0, false};
    CellBits bits = extract_bits<CONF>(L, gray, W, H, quad, P, img, hist);
    if (!bits.ok) return res;
    // border errors (_getBorderErrors) -- number of white bits in the border ring
    const int cells = P.marker_size + 2 * P.marker_border_bits;
    const int bb = P.marker_border_bits, ms = P.marker_size;
    int border_errors = 0;
    for (int y = 0; y < cells; y++)
        for (int x = 0; x < cells; x++) {
            const bool in_border = y < bb || y >= cells - bb || x < bb || x >= cells - bb;
            if (in_border && bits.at(y * cells + x)) border_errors++;
        }
    if constexpr (INV) {
        const int inv_errors = cells * cells - ms * ms - border_errors;  // black bits in the border ring
        if (inv_errors < border_errors) {
            border_errors = inv_errors;
            bits.lo = ~bits.lo;  // bits beyond cells*cells are never read
            bits.hi = ~bits.hi;
            res.inverted = true;
            if constexpr (CONF) {
                const int margin = (int)(P.ignored_margin_per_cell * P.px_per_cell);
                const int win = P.px_per_cell - 2 * margin;
                for (int c = L.lane(); c < cells * cells; c += L.count()) hist[c] = win * win - hist[c];
                L.sync();
            }
        }
    }
    const int max_border = (int)((double)(ms * ms) * P.max_err_border_rate);
    if (border_errors > max_border) return res;
    const unsigned long long cand = inner_code(bits, P);
    const int max_corr = (int)((double)P.max_correction_bits * P.error_correction_rate);
    int first = 0x7fffffff;
    for (int m = L.lane(); m < P.n_markers; m += L.count()) {
        int best = ms * ms + 1, rot = -1;
        for (int r = 0; r < 4; r++) {
            const unsigned long long d = dict[m * 4 + r] ^ cand;
            const int h = fid_popc((uint32_t)d) + fid_popc((uint32_t)(d >> 32));
            if (h < best) {
                best = h;
                rot = r;
            }
        }
        if (best <= max_corr) {
            first = m * 4 + rot;
            break;
        }
    }
    first = L.min_i(first);  // m ascending dominates; rotation rides in the low 2 bits
    if (first != 0x7fffffff) {
        res.id = first >> 2;
        res.rotation = first & 3;
    }
    return res;
}

}  // namespace fid
