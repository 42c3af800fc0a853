// CPU harness for fiducials_b200/csrc/marker_refine.cuh (recovery of missed board markers).  TEST INFRASTRUCTURE ONLY.
// Compiled with g++ by tests/test_hostsim_marker_refine.py into a shared object of its own in a temporary directory, from the same
// header the CUDA kernel k_marker_refine is built from; it is not linked into libfiducials_b200.so.  hs_refine runs the steps of
// k_marker_refine one board after the other, with one lane.
#include <algorithm>
#include <vector>

#include "../../fiducials_b200/csrc/marker_refine.cuh"
#include "../../fiducials_b200/csrc/params_host.h"

using namespace fid;

extern "C" {

// refineDetectedMarkers against n_boards boards in sequence (board b: board_n[b] markers, ids and [.][4][3] object points
// concatenated).  ids / corners ([.][8]) hold n_det detections and receive the recovered ones (capacity max_markers); rej
// [n_rej][8] is the rejected list.  K / D may be NULL.  rec_idx / rec_board [max_markers]: per recovered marker the index into rej as
// passed in and the board; status [n_boards]: 1 the board was refined, 0 nothing to do, -1 cv2 raises (solvePnP, or a board with
// more than one z without a camera).  Returns the number of detections after, or -1 if max_markers is too small.
int hs_refine(const uint8_t* gray, int W, int H, int dictionary, int corner_method, int refine_win, int refine_max_iter, double refine_min_acc,
              double rel_refine_win, float min_rep, float ecr, int check_all, int n_boards, const int32_t* board_n, const int32_t* board_ids,
              const float* board_obj, const double* K, const double* D, int n_det, int32_t* ids, float* corners, int max_markers, int n_rej,
              const float* rej, int32_t* rec_idx, int32_t* rec_board, int32_t* status) {
    fid_params fp;
    default_params(&fp);
    fp.dictionary = dictionary;
    fp.cornerRefinementMethod = corner_method;
    fp.cornerRefinementWinSize = refine_win;
    fp.cornerRefinementMaxIterations = refine_max_iter;
    fp.cornerRefinementMinAccuracy = refine_min_acc;
    fp.relativeCornerRefinmentWinSize = rel_refine_win;
    DevParams P;
    if (make_dev_params(fp, &P) != FID_OK) return -2;
    std::vector<unsigned long long> dict;
    pack_dictionary(P, &dict);
    std::vector<float> masks;
    for (int w = 1; w <= 5; w++) {
        std::vector<float> m((2 * w + 1) * (2 * w + 1));
        subpix_mask(w, m.data());
        masks.insert(masks.end(), m.begin(), m.end());
    }
    const MarkerRefineParams rp{min_rep, ecr, check_all};
    Camera cam{};
    if (K) cam = Camera{K[0], K[4], K[2], K[5], D[0], D[1], D[2], D[3], D[4]};
    const GrayPlane img{gray, (size_t)W};
    const SerialLanes L;
    std::vector<uint8_t> taken(n_rej + 1, 0), scratch(FID_MAX_WARP_SIDE_SQ);
    int hist[256];
    std::vector<float> patch((2 * FID_SUBPIX_MAX_WIN + 3) * (2 * FID_SUBPIX_MAX_WIN + 3));
    int n_taken = 0, n_rec = 0, off = 0;
    for (int b = 0; b < n_boards; b++) {
        const int nb = board_n[b];
        const int32_t* bid = board_ids + off;
        const float* obj = board_obj + (size_t)off * 12;
        off += nb;
        status[b] = 0;
        if (n_det == 0 || n_taken == n_rej) continue;
        std::vector<int32_t> keys(nb), marker_of(nb);
        {
            std::vector<int> ord(nb);
            for (int i = 0; i < nb; i++) ord[i] = i;
            std::sort(ord.begin(), ord.end(), [&](int x, int y) { return bid[x] < bid[y]; });
            for (int i = 0; i < nb; i++) {
                keys[i] = bid[ord[i]];
                marker_of[i] = ord[i];
            }
        }
        // detected board rows (against the detections this call starts with)
        std::vector<int> first(nb, -1);
        for (int j = n_det - 1; j >= 0; j--) {
            const int k = board_find(keys.data(), nb, ids[j]);
            if (k >= 0) first[marker_of[k]] = j;
        }
        double R[9], p[6], Hm[9];
        if (K) {
            std::vector<float> o((size_t)n_det * 12 + 1), ip((size_t)n_det * 8 + 1);
            const int m = board_match(n_det, ids, corners, nb, keys.data(), marker_of.data(), obj, o.data(), ip.data());
            if (m == 0) continue;
            std::vector<double> mn((size_t)m * 8);
            BoardPoseOut po;
            solve_board_pose(4 * m, o.data(), ip.data(), mn.data(), cam, &po);
            if (po.status != 1) {
                status[b] = -1;
                continue;
            }
            for (int k = 0; k < 3; k++) {
                p[k] = po.rvec[k];
                p[3 + k] = po.tvec[k];
            }
            rodrigues_v2m(p, R, nullptr);
        } else {
            bool flat = true;
            for (int i = 0; i < nb * 4; i++) flat = flat && obj[3 * i + 2] == obj[2];
            if (!flat) {
                status[b] = -1;
                continue;
            }
            std::vector<int> rows;
            for (int r = 0; r < nb; r++)
                if (first[r] >= 0) rows.push_back(r);
            if (rows.empty()) continue;
            if (!board_homography((int)rows.size() * 4, [&](int i, float s[2], float d[2]) {
                    const int r = rows[i >> 2], c = i & 3;
                    s[0] = obj[(size_t)r * 12 + 3 * c];
                    s[1] = obj[(size_t)r * 12 + 3 * c + 1];
                    d[0] = corners[(size_t)first[r] * 8 + 2 * c];
                    d[1] = corners[(size_t)first[r] * 8 + 2 * c + 1];
                }, Hm))
                continue;
        }
        status[b] = 1;
        for (int r = 0; r < nb; r++) {
            if (first[r] >= 0) continue;
            float pr[8], q[8];
            if (K) refine_project(obj, r, R, p, cam, pr);
            else refine_transform(obj, r, Hm, pr);
            if (!refine_has_candidate(rp, pr, n_rej, rej, taken.data())) continue;
            const int j = refine_match(L, img, W, H, P, dict.data(), rp, bid[r], pr, n_rej, rej, taken.data(), scratch.data(), hist, q);
            if (j < 0) continue;
            if (n_det >= max_markers) return -1;
            float* out = corners + (size_t)n_det * 8;
            for (int c = 0; c < 4; c++) {
                if (P.corner_refine == 1) refine_subpix_corner(img, W, H, P, masks.data(), q, c, out + 2 * c, patch.data());
                else {
                    out[2 * c] = q[2 * c];
                    out[2 * c + 1] = q[2 * c + 1];
                }
            }
            ids[n_det++] = bid[r];
            taken[j] = 1;
            n_taken++;
            rec_idx[n_rec] = j;
            rec_board[n_rec++] = b;
        }
    }
    return n_det;
}

}  // extern "C"
