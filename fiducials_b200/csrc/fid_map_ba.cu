// fid_map_bundle_adjust: bundle adjustment of a map instance from recorded marker corners on the device (map_ba.cuh states the
// problem, DESIGN.md f16).
//
// Kernels, all double, none with atomics:
//   k_ba_init          warp per candidate frame: its initial pose (map_ba.cuh, ba_init_frame: the board solvePnP, or a marker's own
//                      pose composed with its map pose when that reprojects better)
//   per LM trial step, each kernel returning at once when the run is done or failed:
//     k_ba_eval        thread per observation: its J blocks U, W, V, g and cost (only when a new J is due)
//     k_ba_sums        thread per frame / per free marker: U_f, g_f, cost_f over the frame's observations in detection order,
//                      V_m, g_m over the marker's observations in frame order; the poses of the J
//     k_ba_lm          one thread: the cost summed in frame order, CvLevMarq's bookkeeping (the final pass: rms and sigma^2)
//     k_ba_factor      thread per frame: Cholesky of the damped U_f, h_f = L^-1 g_f
//     k_ba_z           thread per observation of a free marker: Z_o = L_f^-1 W_o
//     k_ba_clear       S = 0, identity rows past 6M
//     k_ba_reduce      warp per nonzero 6x6 block (a <= b) of S: the damped V_a on the diagonal minus sum Z_b^T Z_a over the frames
//                      that see both, in frame order
//     k_ba_rhs         thread per row of S: r = g_m - sum Z^T h over the marker's observations in frame order
//     calib_dense.cuh  the blocked Cholesky of S and the solve of S x = r
//     k_ba_backsub     thread per frame / free marker: x_f = L_f^-T (h_f - sum Z_o x_m), the trial poses and the step norms
//     k_ba_trial       thread per frame: the trial cost over its observations
//     k_ba_decide      one thread: the trial cost and norms summed in frame then marker order, CvLevMarq's accept / reject
//   then the final pass: the undamped S at the optimum factored, diag(S^-1) as |L^-1 e_a|^2 (k_ba_eye + k_dense_trsv by chunks of
//   columns), k_ba_std (thread per free marker: standard deviations and the write-back of its pose into the map).
// The host enqueues one trial step at a time and reads the run's state after it, so nothing is launched once the run is done.
#include "map_ba.cuh"

#include <cuda_runtime.h>
#include <math.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "calib_dense.cuh"
#include "fid_map_internal.h"

#define CKB(call)                                                                                      \
    do {                                                                                               \
        cudaError_t e_ = (call);                                                                       \
        if (e_ != cudaSuccess) {                                                                       \
            fprintf(stderr, "[fiducials_b200] CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); \
            rc = FID_ERR_CUDA;                                                                         \
            goto done;                                                                                 \
        }                                                                                              \
    } while (0)

namespace fid {

#define BA_EYE_COLS 768  // identity columns per chunk of the final pass

struct BaDev {
    int F, M, NO, n6, mp;
    Camera cam;
    const int32_t *f_off, *o_frame, *o_free, *o_slot, *m_off, *m_obs, *free_slot, *b_ab, *b_off, *b_pair;
    const float* o_corner;    // [NO][8]
    const double* slot_obj;   // [slots][4][3]
    double *fpose, *fpose_prev, *spose, *spose_prev;  // [F][12], [slots][12]
    double *blk, *frm, *mrk, *Z, *S, *r, *E, *diag, *fin;  // fin: rms, sigma2
    BaLM* lm;
};

__device__ __forceinline__ bool ba_skip(const BaDev& d, int final_pass, const int* status) {
    return *(volatile const int*)status != 0 || (!final_pass && d.lm->state == 2);
}
__device__ __forceinline__ double ba_scale(const BaDev& d, int final_pass) { return final_pass ? 1.0 : 1.0 + calib_pow10(d.lm->lg); }

__global__ void __launch_bounds__(128) k_ba_init(int nc, const int32_t* c_off, const float* c_obj, const float* c_img, const float* c_len, const double* c_mpose,
                                                 double* c_mn, Camera cam, double* c_pose, int* c_ok) {
    const int c = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (c >= nc) return;
    const int o = c_off[c], n = c_off[c + 1] - o;
    double pose[12];
    const bool ok = ba_init_frame(n, c_obj + 12 * (size_t)o, c_img + 8 * (size_t)o, c_mn + 8 * (size_t)o, cam, c_len + o, c_mpose + 12 * (size_t)o, pose);
    if ((threadIdx.x & 31) == 0) {
        for (int k = 0; k < 12; k++) c_pose[12 * (size_t)c + k] = pose[k];
        c_ok[c] = ok;
    }
}

__global__ void __launch_bounds__(128) k_ba_eval(BaDev d, int final_pass, const int* status) {
    if (ba_skip(d, final_pass, status) || (!final_pass && d.lm->state != 0)) return;
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= d.NO) return;
    const int s = d.o_slot[o];
    ba_obs_eval((const double(*)[3])(d.slot_obj + 12 * (size_t)s), d.o_corner + 8 * (size_t)o, d.cam, d.fpose + 12 * (size_t)d.o_frame[o], d.spose + 12 * (size_t)s,
                d.blk + (size_t)BA_OBS * o);
}

__global__ void __launch_bounds__(128) k_ba_sums(BaDev d, int final_pass, const int* status) {
    if (ba_skip(d, final_pass, status) || (!final_pass && d.lm->state != 0)) return;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < d.F) {
        double q[28];
        for (int k = 0; k < 28; k++) q[k] = 0.0;
        for (int o = d.f_off[i]; o < d.f_off[i + 1]; o++) {
            const double* b = d.blk + (size_t)BA_OBS * o;
            for (int k = 0; k < 21; k++) q[BA_F_U + k] += b[BA_O_U + k];
            for (int k = 0; k < 6; k++) q[BA_F_G + k] += b[BA_O_GF + k];
            q[BA_F_C] += b[BA_O_C];
        }
        for (int k = 0; k < 28; k++) d.frm[(size_t)BA_FRM * i + k] = q[k];
        for (int k = 0; k < 12; k++) d.fpose_prev[12 * (size_t)i + k] = d.fpose[12 * (size_t)i + k];
    } else if (i < d.F + d.M) {
        const int m = i - d.F, s = d.free_slot[m];
        double q[27];
        for (int k = 0; k < 27; k++) q[k] = 0.0;
        for (int t = d.m_off[m]; t < d.m_off[m + 1]; t++) {
            const double* b = d.blk + (size_t)BA_OBS * d.m_obs[t];
            for (int k = 0; k < 21; k++) q[BA_M_V + k] += b[BA_O_V + k];
            for (int k = 0; k < 6; k++) q[BA_M_G + k] += b[BA_O_GM + k];
        }
        for (int k = 0; k < 27; k++) d.mrk[(size_t)BA_MRK * m + k] = q[k];
        for (int k = 0; k < 12; k++) d.spose_prev[12 * (size_t)s + k] = d.spose[12 * (size_t)s + k];
    }
}

__global__ void k_ba_lm(BaDev d, int final_pass, const int* status) {
    if (ba_skip(d, final_pass, status) || (!final_pass && d.lm->state != 0)) return;
    double err = 0.0;
    for (int f = 0; f < d.F; f++) err += d.frm[(size_t)BA_FRM * f + BA_F_C];
    if (final_pass) {
        d.fin[0] = sqrt(err / (4.0 * d.NO));
        d.fin[1] = err / (double)(8LL * d.NO - 6LL * (d.F + d.M));
    } else {
        ba_lm_after_eval(d.lm, err);
    }
}

__global__ void __launch_bounds__(128) k_ba_factor(BaDev d, int final_pass, int* status) {
    if (ba_skip(d, final_pass, status)) return;
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= d.F) return;
    double* q = d.frm + (size_t)BA_FRM * f;
    if (!calib_chol6(q + BA_F_U, ba_scale(d, final_pass), q + BA_F_L)) {
        *status = 1;
        return;
    }
    calib_ro_lsolve6(q + BA_F_L, q + BA_F_G, q + BA_F_H);
}

__global__ void __launch_bounds__(128) k_ba_z(BaDev d, int final_pass, const int* status) {
    if (ba_skip(d, final_pass, status)) return;
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= d.NO || d.o_free[o] < 0) return;
    ba_obs_z(d.frm + (size_t)BA_FRM * d.o_frame[o] + BA_F_L, d.blk + (size_t)BA_OBS * o + BA_O_W, d.Z + 36 * (size_t)o);
}

__global__ void __launch_bounds__(256) k_ba_clear(BaDev d, int final_pass, const int* status) {
    if (ba_skip(d, final_pass, status)) return;
    const size_t n = (size_t)d.mp * d.mp;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (size_t)gridDim.x * blockDim.x) {
        const int a = (int)(e / d.mp), b = (int)(e % d.mp);
        d.S[e] = (a == b && a >= d.n6) ? 1.0 : 0.0;
    }
}

// Warp per block: lanes own entries (i, j) = (e / 6, e % 6), e = lane and lane + 32; rows 6b + i, columns 6a + j.
__global__ void __launch_bounds__(128) k_ba_reduce(BaDev d, int nb, int final_pass, const int* status) {
    if (ba_skip(d, final_pass, status)) return;
    const int k = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (k >= nb) return;
    const int a = d.b_ab[k] & 0xffff, b = (d.b_ab[k] >> 16) & 0xffff;
    const double scale = ba_scale(d, final_pass);
    for (int e = lane; e < 36; e += 32) {
        const int i = e / 6, j = e % 6;
        double s = 0.0;
        if (a == b) {
            const int lo = i < j ? i : j, hi = i < j ? j : i;
            s = d.mrk[(size_t)BA_MRK * a + BA_M_V + lo * 6 - lo * (lo - 1) / 2 + hi - lo];
            if (i == j) s *= scale;
        }
        for (int t = d.b_off[k]; t < d.b_off[k + 1]; t++) {
            const double *za = d.Z + 36 * (size_t)d.b_pair[2 * t], *zb = d.Z + 36 * (size_t)d.b_pair[2 * t + 1];
            double v = 0.0;
            for (int l = 0; l < 6; l++) v += zb[6 * l + i] * za[6 * l + j];
            s -= v;
        }
        d.S[(size_t)(6 * b + i) * d.mp + 6 * a + j] = s;
    }
}

__global__ void __launch_bounds__(128) k_ba_rhs(BaDev d, const int* status) {
    if (ba_skip(d, 0, status)) return;
    const int row = blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= d.mp) return;
    if (row >= d.n6) {
        d.r[row] = 0.0;
        return;
    }
    const int m = row / 6, i = row % 6;
    double s = d.mrk[(size_t)BA_MRK * m + BA_M_G + i];
    for (int t = d.m_off[m]; t < d.m_off[m + 1]; t++) {
        const int o = d.m_obs[t];
        const double *z = d.Z + 36 * (size_t)o, *h = d.frm + (size_t)BA_FRM * d.o_frame[o] + BA_F_H;
        double v = 0.0;
        for (int l = 0; l < 6; l++) v += z[6 * l + i] * h[l];
        s -= v;
    }
    d.r[row] = s;
}

__global__ void __launch_bounds__(128) k_ba_backsub(BaDev d, const int* status) {
    if (ba_skip(d, 0, status)) return;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < d.F) {
        double* q = d.frm + (size_t)BA_FRM * i;
        double y[6], x[6];
        for (int k = 0; k < 6; k++) y[k] = q[BA_F_H + k];
        for (int o = d.f_off[i]; o < d.f_off[i + 1]; o++) {
            if (d.o_free[o] < 0) continue;
            const double *z = d.Z + 36 * (size_t)o, *xm = d.r + 6 * d.o_free[o];
            for (int k = 0; k < 6; k++) {
                double v = 0.0;
                for (int l = 0; l < 6; l++) v += z[6 * k + l] * xm[l];
                y[k] -= v;
            }
        }
        calib_ro_ltsolve6(q + BA_F_L, y, x);
        ba_pose_step(d.fpose_prev + 12 * (size_t)i, x, d.fpose + 12 * (size_t)i, q + BA_F_T + 1);
    } else if (i < d.F + d.M) {
        const int m = i - d.F, s = d.free_slot[m];
        ba_pose_step(d.spose_prev + 12 * (size_t)s, d.r + 6 * m, d.spose + 12 * (size_t)s, d.mrk + (size_t)BA_MRK * m + BA_M_T);
    }
}

__global__ void __launch_bounds__(128) k_ba_trial(BaDev d, const int* status) {
    if (ba_skip(d, 0, status)) return;
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= d.F) return;
    double c = 0.0;
    for (int o = d.f_off[f]; o < d.f_off[f + 1]; o++) {
        const int s = d.o_slot[o];
        c += ba_obs_cost((const double(*)[3])(d.slot_obj + 12 * (size_t)s), d.o_corner + 8 * (size_t)o, d.cam, d.fpose + 12 * (size_t)f, d.spose + 12 * (size_t)s);
    }
    d.frm[(size_t)BA_FRM * f + BA_F_T] = c;
}

__global__ void k_ba_decide(BaDev d, const int* status) {
    if (d.lm->state == 2) return;
    if (*status) {  // a non-positive pivot: the run ends, the call reports it
        d.lm->state = 2;
        return;
    }
    double err = 0.0, dn = 0.0, pn = 0.0;
    for (int f = 0; f < d.F; f++) {
        const double* q = d.frm + (size_t)BA_FRM * f + BA_F_T;
        err += q[0];
        dn += q[1];
        pn += q[2];
    }
    for (int m = 0; m < d.M; m++) {
        dn += d.mrk[(size_t)BA_MRK * m + BA_M_T];
        pn += d.mrk[(size_t)BA_MRK * m + BA_M_T + 1];
    }
    ba_lm_decide(d.lm, err, dn, pn);
}

// Columns a0 .. a0 + ncols - 1 of the identity into E.
__global__ void __launch_bounds__(256) k_ba_eye(BaDev d, int a0, int ncols, const int* status) {
    if (*status) return;
    const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (size_t)ncols * d.mp) return;
    const int c = (int)(e / d.mp), a = (int)(e % d.mp);
    d.E[e] = a == a0 + c ? 1.0 : 0.0;
}

// Thread per free marker: its standard deviations (std [M][6]) and its pose written into the map entry of its slot.
__global__ void __launch_bounds__(128) k_ba_std(BaDev d, MapEntry* entries, double* std_out, const int* status) {
    if (*status) return;
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= d.M) return;
    ba_std(d.diag + 6 * m, d.fin[1], std_out + 6 * (size_t)m);
    const int s = d.free_slot[m];
    for (int k = 0; k < 9; k++) entries[s].pose.R[k] = d.spose[12 * (size_t)s + k];
    for (int k = 0; k < 3; k++) entries[s].pose.t[k] = d.spose[12 * (size_t)s + 9 + k];
}

}  // namespace fid

namespace {

bool finite_camera(const fid_camera* c) {
    for (int k = 0; k < 9; k++)
        if (!std::isfinite(c->K[k])) return false;
    for (int k = 0; k < 5; k++)
        if (!std::isfinite(c->D[k])) return false;
    return c->K[0] > 0 && c->K[4] > 0;
}

}  // namespace

extern "C" int fid_map_ba_default_params(fid_ba_params* p) {
    if (!p) return FID_ERR_INVALID_ARG;
    p->criteria.type = 3;
    p->criteria.max_iter = 100;
    p->criteria.epsilon = 1e-12;
    return FID_OK;
}

extern "C" int fid_map_bundle_adjust(fid_map* m, int instance, int n_frames, const int32_t* counts, const int32_t* ids, const float* corners, int max_markers,
                                     const fid_camera* cam, double fiducial_len, int n_override, const int32_t* override_ids, const double* override_lens,
                                     const fid_ba_params* params, fid_ba_stats* stats, double* frame_rvecs, double* frame_tvecs, int32_t* frame_status,
                                     double* std_entries) {
    using namespace fid;
    if (!m || instance < 0 || instance >= m->p.n_instances || n_frames < 1 || !counts || !ids || !corners || max_markers < 1 || !cam || !finite_camera(cam) ||
        !(fiducial_len > 0) || !std::isfinite(fiducial_len) || n_override < 0 || (n_override > 0 && (!override_ids || !override_lens)))
        return FID_ERR_INVALID_ARG;
    for (int k = 0; k < n_override; k++)
        if (!(override_lens[k] > 0) || !std::isfinite(override_lens[k])) return FID_ERR_INVALID_ARG;
    if (n_frames > BA_MAX_FRAMES) return FID_ERR_CAPACITY;
    for (int f = 0; f < n_frames; f++) {
        if (counts[f] < 0 || counts[f] > max_markers) return FID_ERR_INVALID_ARG;
        const float* c = corners + (size_t)8 * max_markers * f;
        for (int k = 0; k < 8 * counts[f]; k++)
            if (!std::isfinite(c[k])) return FID_ERR_INVALID_ARG;
    }
    int max_iter = 100;
    double eps = 1e-12;
    if (params) {
        if (params->criteria.type & 1) max_iter = std::min(std::max((int)params->criteria.max_iter, 1), 1000);
        if (params->criteria.type & 2) eps = params->criteria.epsilon;
        if (!(eps >= 0) || !std::isfinite(eps)) return FID_ERR_INVALID_ARG;
    }
    CK(cudaSetDevice(m->device));
    CK(cudaStreamSynchronize(m->stream));  // pending asynchronous updates first
    MapState mst;
    CK(cudaMemcpy(&mst, m->d_state + instance, sizeof(mst), cudaMemcpyDeviceToHost));
    const int ns = mst.n, cap = m->p.max_fiducials;
    std::vector<MapEntry> ent(ns);
    if (ns) CK(cudaMemcpy(ent.data(), m->d_entries + (size_t)instance * cap, sizeof(MapEntry) * ns, cudaMemcpyDeviceToHost));
    std::vector<int32_t> slot_ids(ns);
    std::vector<uint8_t> fixed(ns);
    bool any_fixed = false;
    for (int s = 0; s < ns; s++) {
        slot_ids[s] = ent[s].id;
        fixed[s] = ent[s].pose.var == 0.0;
        any_fixed |= fixed[s] != 0;
    }
    if (!any_fixed) return FID_ERR_INVALID_ARG;
    const Camera camera{cam->K[0], cam->K[4], cam->K[2], cam->K[5], cam->D[0], cam->D[1], cam->D[2], cam->D[3], cam->D[4]};
    BaPlan P;
    ba_plan_observations(n_frames, counts, ids, max_markers, ns, slot_ids.data(), &P);
    if (P.c_slot.size() > (size_t)BA_MAX_OBS) return FID_ERR_CAPACITY;
    std::vector<double> slot_obj((size_t)12 * std::max(ns, 1)), spose((size_t)12 * std::max(ns, 1));
    for (int s = 0; s < ns; s++) {
        double o[4][3];
        ba_object_points(ba_marker_len(slot_ids[s], fiducial_len, n_override, override_ids, override_lens), o);
        for (int k = 0; k < 4; k++)
            for (int c = 0; c < 3; c++) slot_obj[12 * s + 3 * k + c] = o[k][c];
        for (int k = 0; k < 9; k++) spose[12 * s + k] = ent[s].pose.R[k];
        for (int k = 0; k < 3; k++) spose[12 * s + 9 + k] = ent[s].pose.t[k];
    }
    const int nc = (int)P.cand.size(), nco = (int)P.c_slot.size();
    int rc = FID_OK, launches = 0, h_status = 0;
    float ms_init = 0.f, ms = 0.f;
    cudaStream_t st = m->stream;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev2 = nullptr, ev3 = nullptr;
    char *mem0 = nullptr, *mem = nullptr;
    std::vector<double> cand_pose((size_t)12 * nc);
    std::vector<int> cand_ok(nc);
    std::vector<uint8_t> init_ok(nc);
    std::vector<double> h_fpose, h_std, h_fin(2);
    BaLM h_lm{};
    int F = 0, M = 0, NO = 0;
    size_t bytes0 = 0, bytes = 0;
    auto carve = [](size_t& total, size_t sz) {
        const size_t at = total;
        total += (sz + 255) & ~(size_t)255;
        return at;
    };
    if (stats) memset(stats, 0, sizeof(*stats));
    CKB(cudaEventCreate(&ev0));
    CKB(cudaEventCreate(&ev1));
    CKB(cudaEventCreate(&ev2));
    CKB(cudaEventCreate(&ev3));
    // ---- stage 1: the initial frame poses ----
    if (nc) {
        std::vector<float> c_obj((size_t)12 * nco), c_img((size_t)8 * nco), c_len(nco);
        std::vector<double> c_mpose((size_t)12 * nco);
        for (int o = 0; o < nco; o++) {
            const int s = P.c_slot[o];
            ba_map_corners(&spose[12 * s], &spose[12 * s + 9], (const double(*)[3]) & slot_obj[12 * s], &c_obj[12 * (size_t)o]);
            memcpy(&c_img[8 * (size_t)o], corners + (size_t)8 * P.c_src[o], sizeof(float) * 8);
            memcpy(&c_mpose[12 * (size_t)o], &spose[12 * s], sizeof(double) * 12);
            c_len[o] = (float)ba_marker_len(slot_ids[s], fiducial_len, n_override, override_ids, override_lens);
        }
        const size_t o_off = carve(bytes0, sizeof(int32_t) * (nc + 1)), o_obj = carve(bytes0, sizeof(float) * c_obj.size()),
                     o_img = carve(bytes0, sizeof(float) * c_img.size()), o_len = carve(bytes0, sizeof(float) * c_len.size()),
                     o_mpose = carve(bytes0, sizeof(double) * c_mpose.size()), o_mn = carve(bytes0, sizeof(double) * 8 * (size_t)nco),
                     o_pose = carve(bytes0, sizeof(double) * cand_pose.size()), o_ok = carve(bytes0, sizeof(int) * nc);
        CKB(cudaMalloc(&mem0, bytes0));
        CKB(cudaEventRecord(ev0, st));
        CKB(cudaMemcpyAsync(mem0 + o_off, P.c_off.data(), sizeof(int32_t) * (nc + 1), cudaMemcpyHostToDevice, st));
        CKB(cudaMemcpyAsync(mem0 + o_obj, c_obj.data(), sizeof(float) * c_obj.size(), cudaMemcpyHostToDevice, st));
        CKB(cudaMemcpyAsync(mem0 + o_img, c_img.data(), sizeof(float) * c_img.size(), cudaMemcpyHostToDevice, st));
        CKB(cudaMemcpyAsync(mem0 + o_len, c_len.data(), sizeof(float) * c_len.size(), cudaMemcpyHostToDevice, st));
        CKB(cudaMemcpyAsync(mem0 + o_mpose, c_mpose.data(), sizeof(double) * c_mpose.size(), cudaMemcpyHostToDevice, st));
        k_ba_init<<<(nc + 3) / 4, 128, 0, st>>>(nc, (const int32_t*)(mem0 + o_off), (const float*)(mem0 + o_obj), (const float*)(mem0 + o_img),
                                                (const float*)(mem0 + o_len), (const double*)(mem0 + o_mpose), (double*)(mem0 + o_mn), camera,
                                                (double*)(mem0 + o_pose), (int*)(mem0 + o_ok));
        launches++;
        CKB(cudaGetLastError());
        CKB(cudaEventRecord(ev1, st));
        CKB(cudaMemcpyAsync(cand_pose.data(), mem0 + o_pose, sizeof(double) * cand_pose.size(), cudaMemcpyDeviceToHost, st));
        CKB(cudaMemcpyAsync(cand_ok.data(), mem0 + o_ok, sizeof(int) * nc, cudaMemcpyDeviceToHost, st));
        CKB(cudaStreamSynchronize(st));
        CKB(cudaEventElapsedTime(&ms_init, ev0, ev1));
        for (int c = 0; c < nc; c++) init_ok[c] = cand_ok[c] != 0;
    }
    ba_plan_solve(ns, fixed.data(), init_ok.data(), &P);
    F = (int)P.frames.size();
    M = P.n_free;
    NO = (int)P.o_slot.size();
    if (stats) {
        stats->frames_used = F;
        stats->markers_used = M;
        stats->observations_used = NO;
        stats->dropped_unmapped = P.n_dropped_unmapped;
        stats->dropped_duplicate = P.n_dropped_duplicate;
        stats->frames_unreached = P.n_unreached_frames;
        stats->markers_unreached = P.n_unreached_markers;
        stats->frames_init_failed = P.n_init_failed;
    }
    if (M > BA_MAX_FREE) {
        rc = FID_ERR_CAPACITY;
        goto done;
    }
    // sigma^2 = sum e^2 / (8 NO - 6 (F + M)) needs no check: every used frame and free marker is joined to a fixed entry by the
    // observations, a bipartite graph over F + M + (fixed) nodes with NO edges, so NO >= F + M and 8 NO > 6 (F + M)
    if (F > 0) {
        // ---- stage 2: the solve ----
        const int n6 = 6 * M, mp = std::max((n6 + DENSE_TILE - 1) / DENSE_TILE * DENSE_TILE, DENSE_TILE), nb = (int)P.b_ab.size();
        const int eye_cols = std::max(std::min(n6, BA_EYE_COLS), 1);
        std::vector<float> o_corner((size_t)8 * NO);
        for (int o = 0; o < NO; o++) memcpy(&o_corner[8 * (size_t)o], corners + (size_t)8 * P.o_src[o], sizeof(float) * 8);
        std::vector<double> fpose((size_t)12 * F);
        for (int f = 0; f < F; f++) memcpy(&fpose[12 * (size_t)f], &cand_pose[12 * (size_t)P.frames[f]], sizeof(double) * 12);
        auto ivec = [&](const std::vector<int32_t>& v) { return carve(bytes, sizeof(int32_t) * std::max<size_t>(v.size(), 1)); };
        const size_t a_foff = ivec(P.f_off), a_oframe = ivec(P.o_frame), a_ofree = ivec(P.o_free), a_oslot = ivec(P.o_slot), a_moff = ivec(P.m_off), a_mobs = ivec(P.m_obs),
                     a_fslot = ivec(P.free_slot), a_bab = ivec(P.b_ab), a_boff = ivec(P.b_off), a_bpair = ivec(P.b_pair),
                     a_corner = carve(bytes, sizeof(float) * o_corner.size()), a_sobj = carve(bytes, sizeof(double) * slot_obj.size()),
                     a_fpose = carve(bytes, sizeof(double) * fpose.size()), a_fprev = carve(bytes, sizeof(double) * fpose.size()),
                     a_spose = carve(bytes, sizeof(double) * spose.size()), a_sprev = carve(bytes, sizeof(double) * spose.size()),
                     a_blk = carve(bytes, sizeof(double) * BA_OBS * (size_t)NO), a_frm = carve(bytes, sizeof(double) * BA_FRM * (size_t)F),
                     a_mrk = carve(bytes, sizeof(double) * BA_MRK * (size_t)std::max(M, 1)), a_Z = carve(bytes, sizeof(double) * 36 * (size_t)NO),
                     a_S = carve(bytes, sizeof(double) * (size_t)mp * mp), a_r = carve(bytes, sizeof(double) * mp), a_E = carve(bytes, sizeof(double) * (size_t)mp * eye_cols),
                     a_diag = carve(bytes, sizeof(double) * mp), a_fin = carve(bytes, sizeof(double) * 2), a_lm = carve(bytes, sizeof(BaLM)),
                     a_status = carve(bytes, sizeof(int)), a_std = carve(bytes, sizeof(double) * 6 * (size_t)std::max(M, 1));
        CKB(cudaMalloc(&mem, bytes));
        BaDev d;
        d.F = F;
        d.M = M;
        d.NO = NO;
        d.n6 = n6;
        d.mp = mp;
        d.cam = camera;
        d.f_off = (const int32_t*)(mem + a_foff);
        d.o_frame = (const int32_t*)(mem + a_oframe);
        d.o_free = (const int32_t*)(mem + a_ofree);
        d.o_slot = (const int32_t*)(mem + a_oslot);
        d.m_off = (const int32_t*)(mem + a_moff);
        d.m_obs = (const int32_t*)(mem + a_mobs);
        d.free_slot = (const int32_t*)(mem + a_fslot);
        d.b_ab = (const int32_t*)(mem + a_bab);
        d.b_off = (const int32_t*)(mem + a_boff);
        d.b_pair = (const int32_t*)(mem + a_bpair);
        d.o_corner = (const float*)(mem + a_corner);
        d.slot_obj = (const double*)(mem + a_sobj);
        d.fpose = (double*)(mem + a_fpose);
        d.fpose_prev = (double*)(mem + a_fprev);
        d.spose = (double*)(mem + a_spose);
        d.spose_prev = (double*)(mem + a_sprev);
        d.blk = (double*)(mem + a_blk);
        d.frm = (double*)(mem + a_frm);
        d.mrk = (double*)(mem + a_mrk);
        d.Z = (double*)(mem + a_Z);
        d.S = (double*)(mem + a_S);
        d.r = (double*)(mem + a_r);
        d.E = (double*)(mem + a_E);
        d.diag = (double*)(mem + a_diag);
        d.fin = (double*)(mem + a_fin);
        d.lm = (BaLM*)(mem + a_lm);
        int* d_status = (int*)(mem + a_status);
        double* d_std = (double*)(mem + a_std);
        BaLM lm0;
        ba_lm_init(&lm0, max_iter, eps);
        auto up = [&](size_t at, const void* src, size_t sz) { return sz ? cudaMemcpyAsync(mem + at, src, sz, cudaMemcpyHostToDevice, st) : cudaSuccess; };
        CKB(cudaEventRecord(ev2, st));
        CKB(up(a_foff, P.f_off.data(), sizeof(int32_t) * P.f_off.size()));
        CKB(up(a_oframe, P.o_frame.data(), sizeof(int32_t) * P.o_frame.size()));
        CKB(up(a_ofree, P.o_free.data(), sizeof(int32_t) * P.o_free.size()));
        CKB(up(a_oslot, P.o_slot.data(), sizeof(int32_t) * P.o_slot.size()));
        CKB(up(a_moff, P.m_off.data(), sizeof(int32_t) * P.m_off.size()));
        CKB(up(a_mobs, P.m_obs.data(), sizeof(int32_t) * P.m_obs.size()));
        CKB(up(a_fslot, P.free_slot.data(), sizeof(int32_t) * P.free_slot.size()));
        CKB(up(a_bab, P.b_ab.data(), sizeof(int32_t) * P.b_ab.size()));
        CKB(up(a_boff, P.b_off.data(), sizeof(int32_t) * P.b_off.size()));
        CKB(up(a_bpair, P.b_pair.data(), sizeof(int32_t) * P.b_pair.size()));
        CKB(up(a_corner, o_corner.data(), sizeof(float) * o_corner.size()));
        CKB(up(a_sobj, slot_obj.data(), sizeof(double) * slot_obj.size()));
        CKB(up(a_fpose, fpose.data(), sizeof(double) * fpose.size()));
        CKB(up(a_spose, spose.data(), sizeof(double) * spose.size()));
        CKB(up(a_lm, &lm0, sizeof(BaLM)));
        CKB(cudaMemsetAsync(d_status, 0, sizeof(int), st));
        {
            const int* state = &d.lm->state;
            const int obs_grid = (NO + 127) / 128, frame_grid = (F + 127) / 128, fm_grid = (F + M + 127) / 128, row_grid = (mp + 127) / 128,
                      block_grid = (nb + 3) / 4, clear_grid = (int)std::min<size_t>(((size_t)mp * mp + 255) / 256, 4096);
            // the reduced system at the J's poses for the run's lambda (final_pass: undamped), factored
            auto reduce = [&](int final_pass) {
                k_ba_factor<<<frame_grid, 128, 0, st>>>(d, final_pass, d_status);
                k_ba_z<<<obs_grid, 128, 0, st>>>(d, final_pass, d_status);
                k_ba_clear<<<clear_grid, 256, 0, st>>>(d, final_pass, d_status);
                launches += 3;
                if (nb > 0) {  // no free marker (every observed entry fixed): S is the padding identity
                    k_ba_reduce<<<block_grid, 128, 0, st>>>(d, nb, final_pass, d_status);
                    launches++;
                }
                if (!final_pass) {
                    k_ba_rhs<<<row_grid, 128, 0, st>>>(d, d_status);
                    launches++;
                }
                launches += dense_cholesky_enqueue(d.S, mp, 1, d_status, final_pass ? nullptr : state, st);
            };
            const int max_steps = BA_MAX_STEPS(max_iter);
            int h_state = 0;
            for (int s = 0; s < max_steps && h_state != 2; s++) {
                k_ba_eval<<<obs_grid, 128, 0, st>>>(d, 0, d_status);
                k_ba_sums<<<fm_grid, 128, 0, st>>>(d, 0, d_status);
                k_ba_lm<<<1, 1, 0, st>>>(d, 0, d_status);
                launches += 3;
                reduce(0);
                k_dense_trsv<<<1, 256, sizeof(double) * mp, st>>>(d.S, mp, mp, d.r, mp, 1, nullptr, d_status, state);
                k_ba_backsub<<<fm_grid, 128, 0, st>>>(d, d_status);
                k_ba_trial<<<frame_grid, 128, 0, st>>>(d, d_status);
                k_ba_decide<<<1, 1, 0, st>>>(d, d_status);
                launches += 4;
                CKB(cudaGetLastError());
                CKB(cudaMemcpyAsync(&h_state, state, sizeof(int), cudaMemcpyDeviceToHost, st));
                CKB(cudaStreamSynchronize(st));
            }
            // final pass: the undamped system at the optimum, diag(S^-1) = |L^-1 e_a|^2
            k_ba_eval<<<obs_grid, 128, 0, st>>>(d, 1, d_status);
            k_ba_sums<<<fm_grid, 128, 0, st>>>(d, 1, d_status);
            k_ba_lm<<<1, 1, 0, st>>>(d, 1, d_status);
            launches += 3;
            reduce(1);
            for (int a0 = 0; a0 < n6; a0 += eye_cols) {
                const int ncols = std::min(n6 - a0, eye_cols);
                k_ba_eye<<<(int)(((size_t)ncols * mp + 255) / 256), 256, 0, st>>>(d, a0, ncols, d_status);
                k_dense_trsv<<<ncols, 256, sizeof(double) * mp, st>>>(d.S, mp, mp, d.E, mp, 0, d.diag + a0, d_status, nullptr);
                launches += 2;
            }
            if (M > 0) {
                k_ba_std<<<(M + 127) / 128, 128, 0, st>>>(d, m->d_entries + (size_t)instance * cap, d_std, d_status);
                launches++;
            }
        }
        CKB(cudaGetLastError());
        CKB(cudaEventRecord(ev3, st));
        h_fpose.resize(fpose.size());
        h_std.resize(6 * (size_t)M);
        CKB(cudaMemcpyAsync(&h_status, d_status, sizeof(int), cudaMemcpyDeviceToHost, st));
        CKB(cudaMemcpyAsync(&h_lm, d.lm, sizeof(BaLM), cudaMemcpyDeviceToHost, st));
        CKB(cudaMemcpyAsync(h_fin.data(), d.fin, sizeof(double) * 2, cudaMemcpyDeviceToHost, st));
        CKB(cudaMemcpyAsync(h_fpose.data(), d.fpose, sizeof(double) * fpose.size(), cudaMemcpyDeviceToHost, st));
        if (M) CKB(cudaMemcpyAsync(h_std.data(), d_std, sizeof(double) * h_std.size(), cudaMemcpyDeviceToHost, st));
        CKB(cudaStreamSynchronize(st));
        CKB(cudaEventElapsedTime(&ms, ev2, ev3));
        if (h_status) {  // a non-positive pivot: nothing was written back (k_ba_std returns at once)
            rc = FID_ERR_INVALID_ARG;
            goto done;
        }
    }
    // outputs
    if (frame_status)
        for (int f = 0; f < n_frames; f++) frame_status[f] = P.status[f];
    if (frame_rvecs) memset(frame_rvecs, 0, sizeof(double) * 3 * (size_t)n_frames);
    if (frame_tvecs) memset(frame_tvecs, 0, sizeof(double) * 3 * (size_t)n_frames);
    for (int f = 0; f < F; f++) {
        const int fi = P.cand[P.frames[f]];
        if (frame_rvecs) rodrigues_m2v(&h_fpose[12 * (size_t)f], frame_rvecs + 3 * (size_t)fi);
        if (frame_tvecs)
            for (int k = 0; k < 3; k++) frame_tvecs[3 * (size_t)fi + k] = h_fpose[12 * (size_t)f + 9 + k];
    }
    if (std_entries) {  // in fid_map_entries order (ascending id)
        std::vector<int> order(ns);
        for (int s = 0; s < ns; s++) order[s] = s;
        std::sort(order.begin(), order.end(), [&](int a, int b) { return slot_ids[a] < slot_ids[b]; });
        for (int k = 0; k < ns; k++) {
            const int fr = F > 0 ? P.slot_free[order[k]] : -1;
            for (int j = 0; j < 6; j++) std_entries[6 * (size_t)k + j] = fr >= 0 ? h_std[6 * (size_t)fr + j] : 0.0;
        }
    }
    if (stats) {
        stats->converged = F > 0 ? h_lm.converged : 1;
        stats->iterations = h_lm.iters;
        stats->n_steps = h_lm.n_steps;
        stats->initial_rms = F > 0 ? sqrt(h_lm.err0 / (4.0 * NO)) : 0.0;
        stats->final_rms = F > 0 ? h_fin[0] : 0.0;
        stats->device_ms = (double)ms_init + (double)ms;
        stats->kernel_launches = launches;
    }
done:
    if (st) cudaStreamSynchronize(st);
    if (mem0) cudaFree(mem0);
    if (mem) cudaFree(mem);
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
    if (ev2) cudaEventDestroy(ev2);
    if (ev3) cudaEventDestroy(ev3);
    return rc;
}
