// fid_calibrate_camera: cv::calibrateCameraExtended on the device (calib.cuh states the computation).
//
// Kernels, all double:
//   k_calib_homography   warp per view: homography and vanishing-point rows (no intrinsic guess)
//   k_calib_init         one warp: the 2x2 normal equations summed in view order, the initial intrinsics
//   k_calib_extrinsics   warp per view: findExtrinsicCameraParams2
//   per LM trial step, each kernel returning at once when the run is done or failed:
//     k_calib_eval       warp per view: U, W, V, gi, ge, cost at the current parameters (only when a new J is due)
//     k_calib_schur      thread per view: Vd^-1 and the view's Schur terms for the current lambda
//     k_calib_solve      one block: the sums of the views in view order (a thread per value), the 9x9 solve
//     k_calib_trial      warp per view: the back-substituted step and the trial cost
//     k_calib_decide     one warp: the trial cost summed in view order, CvLevMarq's accept / reject and lambda
//   then k_calib_eval / k_calib_schur once more at the final parameters (undamped), k_calib_final (one block: S^-1, rms, the
//   intrinsic standard deviations) and k_calib_std (thread per view).
// The host enqueues the <= 2 max_iter + 20 trial steps a run can take and waits once, at the end.
#include "calib.cuh"

#include <cuda_runtime.h>
#include <float.h>
#include <stdio.h>
#include <string.h>

#include <cmath>
#include <vector>

#include "../../include/fiducials_b200.h"

#define CKC(call)                                                                                      \
    do {                                                                                               \
        cudaError_t e_ = (call);                                                                       \
        if (e_ != cudaSuccess) {                                                                       \
            fprintf(stderr, "[fiducials_b200] CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); \
            rc = FID_ERR_CUDA;                                                                         \
            goto done;                                                                                 \
        }                                                                                              \
    } while (0)

namespace fid {

struct CalibDev {
    int nv;
    const int32_t* off;
    const float *obj, *img;
    double *mn, *ab, *init, *p, *pp, *blk, *sch, *trial, *std_ext, *pve;
    CalibLM* lm;
    double* fin;  // rms, sigma2, std_intrinsics[9]
};

__global__ void __launch_bounds__(128) k_calib_homography(CalibDev d, int* status) {
    const int v = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (v >= d.nv) return;
    const int o = d.off[v], n = d.off[v + 1] - o;
    const bool ok = calib_view_homography(n, d.obj + 3 * o, d.img + 2 * o, d.init[2], d.init[3], d.ab + 6 * v);
    if (!ok && (threadIdx.x & 31) == 0) *status = FID_CALIB_E_HOMOGRAPHY;
}

__global__ void k_calib_init(CalibDev d, int width, int height, double aspect, const int* status) {
    __shared__ double t[5];
    if (*status) return;
    const int k = threadIdx.x;
    if (k < 5) {
        double s = 0.0;
        for (int v = 0; v < d.nv; v++) {
            double tv[5];
            calib_view_normal2(d.ab + 6 * v, tv);
            s += tv[k];
        }
        t[k] = s;
    }
    __syncthreads();
    if (k == 0) {
        double A[4];
        calib_init_intrinsics(t, width, height, aspect, A);
        for (int a = 0; a < 4; a++) d.init[a] = A[a];
        for (int a = 4; a < 9; a++) d.init[a] = 0.0;
    }
}

__global__ void __launch_bounds__(128) k_calib_extrinsics(CalibDev d, int* status) {
    const int v = blockIdx.x * 4 + (threadIdx.x >> 5);
    // other warps of this kernel may set *status: one read per warp keeps the warp's board_sum shuffles together
    if (v >= d.nv || __shfl_sync(0xffffffffu, *(volatile const int*)status, 0)) return;
    const int o = d.off[v], n = d.off[v + 1] - o;
    BoardPoseOut out;
    solve_board_pose(n, d.obj + 3 * o, d.img + 2 * o, d.mn + 2 * o, calib_camera(d.init), &out);
    if ((threadIdx.x & 31) == 0) {
        for (int k = 0; k < 3; k++) {
            d.p[6 * v + k] = out.rvec[k];
            d.p[6 * v + 3 + k] = out.tvec[k];
        }
        if (out.status != 1) *status = FID_CALIB_E_EXTRINSICS;
    }
}

__global__ void k_calib_lm_init(CalibDev d, int flags, double aspect, int max_iter, double eps, const int* status) {
    calib_lm_init(d.lm, d.init, flags, aspect, max_iter, eps);
    if (*status) d.lm->state = 2;
}

__global__ void __launch_bounds__(128) k_calib_eval(CalibDev d, int final_pass, const int* status) {
    if (final_pass ? *status != 0 : d.lm->state != 0) return;
    const int v = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (v >= d.nv) return;
    const int o = d.off[v], n = d.off[v + 1] - o;
    double p[6];
    for (int k = 0; k < 6; k++) p[k] = d.p[6 * v + k];
    calib_view_eval(n, d.obj + 3 * o, d.img + 2 * o, d.lm->in, d.lm->aspect, p, d.blk + (size_t)CALIB_BLK * v);
    if ((threadIdx.x & 31) == 0 && !final_pass)
        for (int k = 0; k < 6; k++) d.pp[6 * v + k] = p[k];
}

__global__ void __launch_bounds__(128) k_calib_schur(CalibDev d, int final_pass, const int* status) {
    if (final_pass ? *status != 0 : d.lm->state == 2) return;
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= d.nv) return;
    const double scale = final_pass ? 1.0 : 1.0 + calib_pow10(d.lm->lg);
    calib_view_schur(d.blk + (size_t)CALIB_BLK * v, scale, d.sch + (size_t)CALIB_SCH * v);
}

// Sum of field `base + k` of every view's record (stride doubles), in view order.
__device__ double calib_sum_views(const double* a, int nv, size_t stride, int k) {
    double s = 0.0;
    for (int v = 0; v < nv; v++) s += a[stride * v + k];
    return s;
}

__global__ void __launch_bounds__(128) k_calib_solve(CalibDev d) {
    __shared__ double Q[45], q[9];
    CalibLM* lm = d.lm;
    const int state = lm->state;
    if (state == 2) return;
    const int k = threadIdx.x;
    if (state == 0) {  // a new J: the sums of U, gi and the cost
        if (k < 45) lm->U[k] = calib_sum_views(d.blk, d.nv, CALIB_BLK, CALIB_U + k);
        else if (k < 54) lm->g[k - 45] = calib_sum_views(d.blk, d.nv, CALIB_BLK, CALIB_GI + k - 45);
        else if (k == 54) lm->err = calib_sum_views(d.blk, d.nv, CALIB_BLK, CALIB_COST);
    }
    if (k < 45) Q[k] = calib_sum_views(d.sch, d.nv, CALIB_SCH, CALIB_Q + k);
    else if (k < 54) q[k - 45] = calib_sum_views(d.sch, d.nv, CALIB_SCH, CALIB_QV + k - 45);
    __syncthreads();
    if (k == 0) {
        if (state == 0) {
            calib_lm_after_eval(lm, lm->err);
            lm->state = 1;
        }
        double dint[9];
        calib_solve_intrinsics(lm->U, lm->g, Q, q, 1.0 + calib_pow10(lm->lg), lm->mask, dint);
        calib_lm_trial_intrinsics(lm, dint);
    }
}

__global__ void __launch_bounds__(128) k_calib_trial(CalibDev d) {
    if (d.lm->state == 2) return;
    const int v = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (v >= d.nv) return;
    const int o = d.off[v], n = d.off[v + 1] - o;
    double pp[6], p[6], out[3];
    for (int k = 0; k < 6; k++) pp[k] = d.pp[6 * v + k];
    calib_view_trial(n, d.obj + 3 * o, d.img + 2 * o, d.lm->in, d.lm->aspect, d.blk + (size_t)CALIB_BLK * v, d.sch + (size_t)CALIB_SCH * v, d.lm->dint, pp, p,
                     out);
    if ((threadIdx.x & 31) == 0) {
        for (int k = 0; k < 6; k++) d.p[6 * v + k] = p[k];
        for (int k = 0; k < 3; k++) d.trial[3 * v + k] = out[k];
    }
}

__global__ void k_calib_decide(CalibDev d) {
    __shared__ double t[3];
    if (d.lm->state == 2) return;
    const int k = threadIdx.x;
    if (k < 3) t[k] = calib_sum_views(d.trial, d.nv, 3, k);
    __syncthreads();
    if (k == 0) calib_lm_decide(d.lm, t[0], t[1], t[2]);
}

__global__ void __launch_bounds__(128) k_calib_final(CalibDev d, int total, const int* status) {
    __shared__ double U[45], Q[45], err;
    if (*status) return;
    const int k = threadIdx.x;
    if (k < 45) {
        U[k] = calib_sum_views(d.blk, d.nv, CALIB_BLK, CALIB_U + k);
        Q[k] = calib_sum_views(d.sch, d.nv, CALIB_SCH, CALIB_Q + k);
    } else if (k == 45) {
        err = calib_sum_views(d.blk, d.nv, CALIB_BLK, CALIB_COST);
    }
    __syncthreads();
    if (k == 0) {
        CalibLM* lm = d.lm;
        lm->n_evals++;
        double Sinv[9][9];
        calib_schur_inverse(U, Q, lm->mask, Sinv);
        int nfree = 6 * d.nv;
        for (int a = 0; a < 9; a++) nfree += lm->mask[a];
        const double sigma2 = err / (double)(2 * total - nfree);
        d.fin[0] = sqrt(err / total);
        d.fin[1] = sigma2;
        for (int a = 0; a < 9; a++) d.fin[2 + a] = lm->mask[a] ? sqrt(Sinv[a][a] * sigma2) : 0.0;
        for (int a = 0; a < 81; a++) d.fin[11 + a] = Sinv[a / 9][a % 9];
    }
}

__global__ void __launch_bounds__(128) k_calib_std(CalibDev d, const int* status) {
    if (*status) return;
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= d.nv) return;
    double Sinv[9][9];
    for (int a = 0; a < 81; a++) Sinv[a / 9][a % 9] = d.fin[11 + a];
    calib_view_std(d.blk + (size_t)CALIB_BLK * v, d.sch + (size_t)CALIB_SCH * v, Sinv, d.fin[1], d.std_ext + 6 * v);
    d.pve[v] = sqrt(d.blk[(size_t)CALIB_BLK * v + CALIB_COST] / (d.off[v + 1] - d.off[v]));
}

}  // namespace fid

namespace {

// What fid_calibrate_camera and fid_calibrate_camera_ro check and derive before any device work.
struct CalibInput {
    int total, max_iter;
    double eps, aspect;
    bool use_guess;
    fid_camera g;
    std::vector<float> objz;  // obj with z = 0 for a planar rig without a guess
};

// The checks where cv2 raises, CvLevMarq's criteria and the guess: FID_OK, FID_ERR_UNSUPPORTED, or a FID_CALIB_E_* status (> 0).
int calib_check(int n_views, const int32_t* offsets, const float* obj, const float* img, int width, int height, const fid_camera* guess, int32_t flags,
                const fid_calib_criteria* criteria, CalibInput* ci) {
    const int supported = FID_CALIB_USE_INTRINSIC_GUESS | FID_CALIB_FIX_ASPECT_RATIO | FID_CALIB_FIX_PRINCIPAL_POINT | FID_CALIB_ZERO_TANGENT_DIST |
                          FID_CALIB_FIX_FOCAL_LENGTH | FID_CALIB_FIX_K1 | FID_CALIB_FIX_K2 | FID_CALIB_FIX_K3;
    if (flags & ~supported) return FID_ERR_UNSUPPORTED;
    if (n_views < 1 || n_views > FID_CALIB_MAX_VIEWS || !offsets || !obj || !img || width < 1 || height < 1 || offsets[0] != 0) return FID_CALIB_E_INPUT;
    for (int v = 0; v < n_views; v++) {
        const int n = offsets[v + 1] - offsets[v];
        if (offsets[v + 1] < offsets[v] || offsets[v + 1] > FID_CALIB_MAX_TOTAL) return FID_CALIB_E_INPUT;
        if (n < 4 || n > FID_CALIB_MAX_POINTS) return FID_CALIB_E_POINTS;
    }
    const int total = offsets[n_views];
    ci->total = total;
    for (size_t i = 0; i < (size_t)total * 3; i++)
        if (!std::isfinite(obj[i])) return FID_CALIB_E_INPUT;
    for (size_t i = 0; i < (size_t)total * 2; i++)
        if (!std::isfinite(img[i])) return FID_CALIB_E_INPUT;
    // CvLevMarq's criteria
    ci->max_iter = 30;
    ci->eps = DBL_EPSILON;
    if (criteria) {
        if (criteria->type & 1) ci->max_iter = criteria->max_iter < 1 ? 1 : (criteria->max_iter > 1000 ? 1000 : criteria->max_iter);
        if (criteria->type & 2) {
            if (std::isnan(criteria->epsilon)) return FID_CALIB_E_INPUT;
            ci->eps = criteria->epsilon > 0 ? criteria->epsilon : 0.0;
        }
    }
    fid_camera& g = ci->g;
    memset(&g, 0, sizeof(g));
    g.K[0] = g.K[4] = g.K[8] = 1.0;
    if (guess) g = *guess;
    else if (flags & FID_CALIB_USE_INTRINSIC_GUESS) return FID_CALIB_E_GUESS;
    for (int k = 0; k < 9; k++)
        if (!std::isfinite(g.K[k]) || (k < 5 && !std::isfinite(g.D[k]))) return FID_CALIB_E_INPUT;
    ci->use_guess = flags & FID_CALIB_USE_INTRINSIC_GUESS;
    if (ci->use_guess) {
        const double* K = g.K;
        if (K[0] <= 0 || K[4] <= 0 || K[2] < 0 || K[2] >= width || K[5] < 0 || K[5] >= height || fabs(K[1]) > 1e-5 || fabs(K[3]) > 1e-5 || fabs(K[6]) > 1e-5 ||
            fabs(K[7]) > 1e-5 || fabs(K[8] - 1) > 1e-5)
            return FID_CALIB_E_GUESS;
    }
    ci->aspect = 0.0;
    if (flags & FID_CALIB_FIX_ASPECT_RATIO) {
        ci->aspect = g.K[0] / g.K[4];
        if (!(ci->aspect >= 0.01 && ci->aspect <= 100.0)) return FID_CALIB_E_GUESS;
    }
    ci->objz.assign(obj, obj + (size_t)total * 3);
    if (!ci->use_guess) {  // planar rigs only: meanStdDev of z, then z = 0
        double s = 0.0, sq = 0.0;
        for (int i = 0; i < total; i++) {
            const double z = obj[3 * i + 2];
            s += z;
            sq += z * z;
        }
        const double mean = s / total, var = sq / total - mean * mean, sdv = sqrt(var > 0 ? var : 0.0);
        if (fabs(mean) > 1e-5 || sdv > 1e-5) return FID_CALIB_E_NONPLANAR;
        for (int i = 0; i < total; i++) ci->objz[3 * i + 2] = 0.0f;
    }
    return FID_OK;
}

// The outputs both calls return from the device's final state: fin = rms, sigma2, std_intrinsics[9]; p, std, pve per view.
void calib_fill_result(const fid::CalibLM* lm, const double* fin, const std::vector<double>& p, const std::vector<double>& std, const std::vector<double>& pve,
                       int nv, fid_calib_result* result, double* rvecs, double* tvecs, double* std_extrinsics, double* per_view_errors) {
    result->rms = fin[0];
    memset(&result->camera, 0, sizeof(result->camera));
    result->camera.K[0] = lm->in[0];
    result->camera.K[2] = lm->in[2];
    result->camera.K[4] = lm->in[1];
    result->camera.K[5] = lm->in[3];
    result->camera.K[8] = 1.0;
    for (int k = 0; k < 5; k++) result->camera.D[k] = lm->in[4 + k];
    for (int a = 0; a < 9; a++) result->std_intrinsics[a] = fin[2 + a];
    result->iterations = lm->iters;
    for (int v = 0; v < nv; v++)
        for (int k = 0; k < 3; k++) {
            if (rvecs) rvecs[3 * v + k] = p[6 * v + k];
            if (tvecs) tvecs[3 * v + k] = p[6 * v + 3 + k];
        }
    if (std_extrinsics) memcpy(std_extrinsics, std.data(), sizeof(double) * 6 * nv);
    if (per_view_errors) memcpy(per_view_errors, pve.data(), sizeof(double) * nv);
}

void calib_fill_stats(const fid::CalibLM* lm, int launches, float ms, fid_calib_stats* stats) {
    if (!stats) return;
    stats->n_steps = lm->n_steps;
    stats->n_evaluations = lm->n_evals;
    stats->kernel_launches = launches;
    stats->device_ms = ms;
    memcpy(stats->steps, lm->steps, lm->n_steps < FID_CALIB_MAX_STEPS ? lm->n_steps : FID_CALIB_MAX_STEPS);
}

}  // namespace

extern "C" int fid_calibrate_camera(int device, int n_views, const int32_t* offsets, const float* obj, const float* img, int width, int height, const fid_camera* guess,
                                    int32_t flags, const fid_calib_criteria* criteria, fid_calib_result* result, double* rvecs, double* tvecs, double* std_extrinsics,
                                    double* per_view_errors, fid_calib_stats* stats) {
    using namespace fid;
    if (!result) return FID_ERR_INVALID_ARG;
    memset(result, 0, sizeof(*result));
    if (stats) memset(stats, 0, sizeof(*stats));
    auto fail = [&](int why) {
        result->status = why;
        return FID_ERR_INVALID_ARG;
    };
    CalibInput ci;
    const int chk = calib_check(n_views, offsets, obj, img, width, height, guess, flags, criteria, &ci);
    if (chk < 0) return chk;
    if (chk > 0) return fail(chk);
    const int total = ci.total, max_iter = ci.max_iter;
    const double eps = ci.eps, aspect = ci.aspect;
    const bool use_guess = ci.use_guess;
    const fid_camera& g = ci.g;
    const std::vector<float>& objz = ci.objz;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) {
        cudaGetLastError();
        return FID_ERR_NO_DEVICE;
    }
    int prev_device = 0;
    cudaGetDevice(&prev_device);
    int rc = FID_OK, launches = 0, h_status = 0;
    cudaStream_t st = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    char* mem = nullptr;
    const int nv = n_views;
    CalibDev d;
    std::vector<char> lm_buf(sizeof(CalibLM));
    CalibLM* h_lm = (CalibLM*)lm_buf.data();
    double init[9];  // the initial intrinsics: the guess, or the principal point of initIntrinsicParams2D
    if (use_guess) {
        const double A[9] = {g.K[0], g.K[4], g.K[2], g.K[5], g.D[0], g.D[1], g.D[2], g.D[3], g.D[4]};
        memcpy(init, A, sizeof(init));
    } else {
        const double A[9] = {0, 0, (width - 1) * 0.5, (height - 1) * 0.5, 0, 0, 0, 0, 0};
        memcpy(init, A, sizeof(init));
    }
    std::vector<double> h_p, h_std, h_pve, h_fin(92);
    float ms = 0.0f;
    size_t bytes = 0;
    const size_t sz_off = sizeof(int32_t) * (nv + 1), sz_obj = sizeof(float) * 3 * (size_t)total, sz_img = sizeof(float) * 2 * (size_t)total;
    auto carve = [&](size_t n) {
        const size_t at = bytes;
        bytes += (n + 255) & ~(size_t)255;
        return at;
    };
    const size_t o_off = carve(sz_off), o_obj = carve(sz_obj), o_img = carve(sz_img), o_mn = carve(sizeof(double) * 2 * (size_t)total),
                 o_ab = carve(sizeof(double) * 6 * nv), o_init = carve(sizeof(double) * 9), o_p = carve(sizeof(double) * 6 * nv),
                 o_pp = carve(sizeof(double) * 6 * nv), o_blk = carve(sizeof(double) * CALIB_BLK * (size_t)nv), o_sch = carve(sizeof(double) * CALIB_SCH * (size_t)nv),
                 o_trial = carve(sizeof(double) * 3 * nv), o_std = carve(sizeof(double) * 6 * nv), o_pve = carve(sizeof(double) * nv),
                 o_lm = carve(sizeof(CalibLM)), o_fin = carve(sizeof(double) * 92), o_status = carve(sizeof(int));
    const int warp_grid = (nv + 3) / 4, thread_grid = (nv + 127) / 128;
    const int max_steps = 2 * max_iter + 20;
    int* d_status;
    CKC(cudaSetDevice(device));
    CKC(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    CKC(cudaEventCreate(&ev0));
    CKC(cudaEventCreate(&ev1));
    CKC(cudaMalloc(&mem, bytes));
    d.nv = nv;
    d.off = (const int32_t*)(mem + o_off);
    d.obj = (const float*)(mem + o_obj);
    d.img = (const float*)(mem + o_img);
    d.mn = (double*)(mem + o_mn);
    d.ab = (double*)(mem + o_ab);
    d.init = (double*)(mem + o_init);
    d.p = (double*)(mem + o_p);
    d.pp = (double*)(mem + o_pp);
    d.blk = (double*)(mem + o_blk);
    d.sch = (double*)(mem + o_sch);
    d.trial = (double*)(mem + o_trial);
    d.std_ext = (double*)(mem + o_std);
    d.pve = (double*)(mem + o_pve);
    d.lm = (CalibLM*)(mem + o_lm);
    d.fin = (double*)(mem + o_fin);
    d_status = (int*)(mem + o_status);
    CKC(cudaEventRecord(ev0, st));
    CKC(cudaMemcpyAsync(mem + o_off, offsets, sz_off, cudaMemcpyHostToDevice, st));
    CKC(cudaMemcpyAsync(mem + o_obj, objz.data(), sz_obj, cudaMemcpyHostToDevice, st));
    CKC(cudaMemcpyAsync(mem + o_img, img, sz_img, cudaMemcpyHostToDevice, st));
    CKC(cudaMemsetAsync(d_status, 0, sizeof(int), st));
    CKC(cudaMemcpyAsync(d.init, init, sizeof(init), cudaMemcpyHostToDevice, st));
    if (!use_guess) {
        k_calib_homography<<<warp_grid, 128, 0, st>>>(d, d_status);
        k_calib_init<<<1, 32, 0, st>>>(d, width, height, aspect, d_status);
        launches += 2;
    }
    k_calib_extrinsics<<<warp_grid, 128, 0, st>>>(d, d_status);
    k_calib_lm_init<<<1, 1, 0, st>>>(d, flags, aspect, max_iter, eps, d_status);
    launches += 2;
    for (int s = 0; s < max_steps; s++) {
        k_calib_eval<<<warp_grid, 128, 0, st>>>(d, 0, d_status);
        k_calib_schur<<<thread_grid, 128, 0, st>>>(d, 0, d_status);
        k_calib_solve<<<1, 128, 0, st>>>(d);
        k_calib_trial<<<warp_grid, 128, 0, st>>>(d);
        k_calib_decide<<<1, 32, 0, st>>>(d);
        launches += 5;
    }
    k_calib_eval<<<warp_grid, 128, 0, st>>>(d, 1, d_status);
    k_calib_schur<<<thread_grid, 128, 0, st>>>(d, 1, d_status);
    k_calib_final<<<1, 128, 0, st>>>(d, total, d_status);
    k_calib_std<<<thread_grid, 128, 0, st>>>(d, d_status);
    launches += 4;
    CKC(cudaGetLastError());
    CKC(cudaEventRecord(ev1, st));
    h_p.resize(6 * (size_t)nv);
    h_std.resize(6 * (size_t)nv);
    h_pve.resize(nv);
    CKC(cudaMemcpyAsync(&h_status, d_status, sizeof(int), cudaMemcpyDeviceToHost, st));
    CKC(cudaMemcpyAsync(h_lm, d.lm, sizeof(CalibLM), cudaMemcpyDeviceToHost, st));
    CKC(cudaMemcpyAsync(h_p.data(), d.p, sizeof(double) * 6 * nv, cudaMemcpyDeviceToHost, st));
    CKC(cudaMemcpyAsync(h_std.data(), d.std_ext, sizeof(double) * 6 * nv, cudaMemcpyDeviceToHost, st));
    CKC(cudaMemcpyAsync(h_pve.data(), d.pve, sizeof(double) * nv, cudaMemcpyDeviceToHost, st));
    CKC(cudaMemcpyAsync(h_fin.data(), d.fin, sizeof(double) * 92, cudaMemcpyDeviceToHost, st));
    CKC(cudaStreamSynchronize(st));
    CKC(cudaEventElapsedTime(&ms, ev0, ev1));
    if (h_status) {
        rc = fail(h_status);
        goto done;
    }
    calib_fill_result(h_lm, h_fin.data(), h_p, h_std, h_pve, nv, result, rvecs, tvecs, std_extrinsics, per_view_errors);
    calib_fill_stats(h_lm, launches, ms, stats);
done:
    if (st) cudaStreamSynchronize(st);
    if (mem) cudaFree(mem);
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
    if (st) cudaStreamDestroy(st);
    cudaSetDevice(prev_device);
    return rc;
}

// ---- fid_calibrate_camera_ro: object release (calib.cuh, "object release"; the dense kernels are calib_dense.cuh's) -----------
//   before the LM: k_calib_homography / k_calib_init (no guess), k_calib_extrinsics, k_calib_lm_init, as fid_calibrate_camera
//   per LM trial step, each kernel returning at once when the run is done or failed:
//     k_ro_eval       warp per view: U, W, V, gi, ge, cost at the board's current points (only when a new J is due)
//     k_ro_points     thread per point: the point's sums over the views in view order (only when a new J is due)
//     k_ro_sums       one block: the sums of U, gi and the cost in view order, CvLevMarq's bookkeeping of a new J
//     k_ro_factor     thread per view: L of the damped V and h = L^-1 ge
//     k_ro_init       thread per entry: A (damped) and g over the padded system
//     per chunk of <= 256 views: k_ro_zbuild (Z^T of the chunk), k_ro_rhs (r -= Z h in view order), k_dense_syrk (S -= Z Z^T)
//     the blocked Cholesky (3 launches per 32 columns), k_dense_trsv (the step), k_ro_step (trial intrinsics and board),
//     k_ro_trial (warp per view: back-substitution and trial cost), k_ro_decide (CvLevMarq's accept / reject)
//   then the undamped system at the final parameters, factored as above; per chunk k_ro_zbuild, k_dense_trsv (T = L^-1 Z) and
//   k_ro_view_std; per chunk of identity columns k_ro_eye and k_dense_trsv (diag S^-1 as |L^-1 e_a|^2); k_ro_final.
#include "calib_dense.cuh"

namespace fid {

#define CALIB_RO_CHUNK 256  // views per chunk of Z

struct CalibRoDev {
    CalibDev c;
    int n, fixed, m, mp, cols;  // points per view, fixed point, 9 + 3n, padded to 32, columns of the Z buffer
    double *board, *board_prev, *pts, *fac, *S, *r, *Z, *diag, *on, *std_obj;
};

__device__ __forceinline__ bool ro_skip(const CalibRoDev& d, int final_pass, const int* status) { return *status != 0 || (!final_pass && d.c.lm->state == 2); }

__global__ void __launch_bounds__(128) k_ro_eval(CalibRoDev d, int final_pass, const int* status) {
    if (ro_skip(d, final_pass, status) || (!final_pass && d.c.lm->state != 0)) return;
    const int v = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (v >= d.c.nv) return;
    double p[6];
    for (int k = 0; k < 6; k++) p[k] = d.c.p[6 * v + k];
    calib_view_eval(d.n, d.board, d.c.img + 2 * (size_t)d.n * v, d.c.lm->in, d.c.lm->aspect, p, d.c.blk + (size_t)CALIB_BLK * v);
    if ((threadIdx.x & 31) == 0 && !final_pass)
        for (int k = 0; k < 6; k++) d.c.pp[6 * v + k] = p[k];
}

__global__ void __launch_bounds__(128) k_ro_points(CalibRoDev d, int final_pass, const int* status) {
    if (ro_skip(d, final_pass, status) || (!final_pass && d.c.lm->state != 0)) return;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= d.n) return;
    calib_ro_point_sums(d.c.nv, d.n, i, d.board, d.c.img, d.c.lm->in, d.c.lm->aspect, d.c.p, d.pts + (size_t)CALIB_PT * i);
    if (!final_pass)
        for (int c = 0; c < 3; c++) d.board_prev[3 * i + c] = d.board[3 * i + c];
}

// fin: rms, sigma2 (final pass)
__global__ void __launch_bounds__(64) k_ro_sums(CalibRoDev d, int final_pass, const int* status) {
    if (ro_skip(d, final_pass, status)) return;
    CalibLM* lm = d.c.lm;
    if (!final_pass && lm->state != 0) return;
    __shared__ double err;
    const int k = threadIdx.x;
    if (k < 45) lm->U[k] = calib_sum_views(d.c.blk, d.c.nv, CALIB_BLK, CALIB_U + k);
    else if (k < 54) lm->g[k - 45] = calib_sum_views(d.c.blk, d.c.nv, CALIB_BLK, CALIB_GI + k - 45);
    else if (k == 54) err = calib_sum_views(d.c.blk, d.c.nv, CALIB_BLK, CALIB_COST);
    __syncthreads();
    if (k != 0) return;
    if (final_pass) {
        lm->n_evals++;
        const int total = d.n * d.c.nv;
        d.c.fin[0] = sqrt(err / total);
        d.c.fin[1] = err / (double)(2 * total - calib_ro_nfree(lm->mask, d.c.nv, d.n));
    } else {
        lm->err = err;
        calib_lm_after_eval(lm, err);
        lm->state = 1;
    }
}

__global__ void __launch_bounds__(128) k_ro_factor(CalibRoDev d, int final_pass, int* status) {
    if (ro_skip(d, final_pass, status)) return;
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= d.c.nv) return;
    const double scale = final_pass ? 1.0 : 1.0 + calib_pow10(d.c.lm->lg);
    if (!calib_ro_view_factor(d.c.blk + (size_t)CALIB_BLK * v, scale, d.fac + (size_t)CALIB_FAC * v)) *status = FID_CALIB_E_RO_SINGULAR;
}

// Grid (mp / 32, mp / 8) of (32, 8) threads: S's lower triangle from A, and r = g.
__global__ void __launch_bounds__(256) k_ro_init(CalibRoDev d, int final_pass, const int* status) {
    if (ro_skip(d, final_pass, status)) return;
    const int b = blockIdx.x * 32 + threadIdx.x, a = blockIdx.y * 8 + threadIdx.y;
    if (a >= d.mp || b > a) return;
    const CalibLM* lm = d.c.lm;
    const double scale = final_pass ? 1.0 : 1.0 + calib_pow10(lm->lg);
    d.S[(size_t)a * d.mp + b] = calib_ro_entry(a, b, d.n, d.fixed, lm->mask, lm->U, d.pts, scale);
    if (b == 0) d.r[a] = calib_ro_grad(a, d.n, d.fixed, lm->mask, lm->g, d.pts);
}

// Grid ((n + 128) / 128, views of the chunk): Z^T of views v0.. (column 6 (v - v0) + j, length mp) at the J's parameters
// (the last accepted ones in a step, the final ones in the final pass).
__global__ void __launch_bounds__(128) k_ro_zbuild(CalibRoDev d, int v0, int final_pass, const int* status) {
    if (ro_skip(d, final_pass, status)) return;
    const int t = blockIdx.x * blockDim.x + threadIdx.x, vv = blockIdx.y, v = v0 + vv;
    if (t > d.n) return;
    const CalibLM* lm = d.c.lm;
    const double* fac = d.fac + (size_t)CALIB_FAC * v;
    double* col = d.Z + (size_t)6 * vv * d.mp;
    if (t < d.n) {
        double z[3][6];
        calib_ro_z_point((final_pass ? d.board : d.board_prev) + 3 * t, d.c.img + 2 * ((size_t)d.n * v + t), final_pass ? lm->in : lm->in_prev, lm->aspect,
                         (final_pass ? d.c.p : d.c.pp) + 6 * v, fac, t, d.n, d.fixed, z);
        for (int c = 0; c < 3; c++)
            for (int j = 0; j < 6; j++) col[(size_t)j * d.mp + 9 + 3 * t + c] = z[c][j];
    } else {
        double z[9][6];
        calib_ro_z_intrinsics(d.c.blk + (size_t)CALIB_BLK * v, fac, lm->mask, z);
        for (int a = 0; a < 9; a++)
            for (int j = 0; j < 6; j++) col[(size_t)j * d.mp + a] = z[a][j];
    }
}

// Thread per row: r -= Z_v h_v for the views v0 .. v0 + nvc - 1, in view order.
__global__ void __launch_bounds__(128) k_ro_rhs(CalibRoDev d, int v0, int nvc, const int* status) {
    if (ro_skip(d, 0, status)) return;
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= d.mp) return;
    double r = d.r[a];
    for (int vv = 0; vv < nvc; vv++) {
        const double* h = d.fac + (size_t)CALIB_FAC * (v0 + vv) + CALIB_FAC_H;
        double s = 0.0;
        for (int j = 0; j < 6; j++) s += d.Z[((size_t)6 * vv + j) * d.mp + a] * h[j];
        r -= s;
    }
    d.r[a] = r;
}

__global__ void k_ro_step(CalibRoDev d, const int* status) {
    if (ro_skip(d, 0, status)) return;
    calib_lm_trial_intrinsics(d.c.lm, d.r);
    calib_ro_obj_trial(d.n, d.fixed, d.board_prev, d.r + 9, d.board, d.on);
}

__global__ void __launch_bounds__(128) k_ro_trial(CalibRoDev d, const int* status) {
    if (ro_skip(d, 0, status)) return;
    const int v = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (v >= d.c.nv) return;
    const CalibLM* lm = d.c.lm;
    double pp[6], p[6], out[3];
    for (int k = 0; k < 6; k++) pp[k] = d.c.pp[6 * v + k];
    calib_ro_view_trial(d.n, d.board_prev, d.board, d.r + 9, d.c.img + 2 * (size_t)d.n * v, lm->in_prev, lm->in, lm->aspect, d.c.blk + (size_t)CALIB_BLK * v,
                        d.fac + (size_t)CALIB_FAC * v, lm->dint, pp, p, out);
    if ((threadIdx.x & 31) == 0) {
        for (int k = 0; k < 6; k++) d.c.p[6 * v + k] = p[k];
        for (int k = 0; k < 3; k++) d.c.trial[3 * v + k] = out[k];
    }
}

__global__ void k_ro_decide(CalibRoDev d, const int* status) {
    __shared__ double t[3];
    CalibLM* lm = d.c.lm;
    if (lm->state == 2) return;
    if (*status) {  // a non-positive pivot: the run ends, the call reports it
        if (threadIdx.x == 0) lm->state = 2;
        return;
    }
    const int k = threadIdx.x;
    if (k < 3) t[k] = calib_sum_views(d.c.trial, d.c.nv, 3, k);
    __syncthreads();
    if (k == 0) calib_lm_decide(lm, t[0], t[1] + d.on[0], t[2] + d.on[1]);
}

// Thread per view of the chunk: M = T^T T (T = L_S^-1 Z, the chunk's columns after the forward solve), the view's standard
// deviations and its error.
__global__ void __launch_bounds__(128) k_ro_view_std(CalibRoDev d, int v0, int nvc, const int* status) {
    if (*status) return;
    const int vv = blockIdx.x * blockDim.x + threadIdx.x, v = v0 + vv;
    if (vv >= nvc) return;
    const double* T = d.Z + (size_t)6 * vv * d.mp;
    double M[36];
    for (int j = 0; j < 6; j++)
        for (int k = 0; k < 6; k++) {
            double s = 0.0;
            for (int a = 0; a < d.mp; a++) s += T[(size_t)j * d.mp + a] * T[(size_t)k * d.mp + a];
            M[6 * j + k] = s;
        }
    calib_ro_view_std(d.fac + (size_t)CALIB_FAC * v, M, d.c.fin[1], d.c.std_ext + 6 * v);
    d.c.pve[v] = sqrt(d.c.blk[(size_t)CALIB_BLK * v + CALIB_COST] / d.n);
}

// Columns a0 .. a0 + ncols - 1 of the identity into the Z buffer.
__global__ void __launch_bounds__(256) k_ro_eye(CalibRoDev d, int a0, int ncols, const int* status) {
    if (*status) return;
    const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (size_t)ncols * d.mp) return;
    const int c = (int)(e / d.mp), a = (int)(e % d.mp);
    d.Z[e] = a == a0 + c ? 1.0 : 0.0;
}

// The standard deviations of the intrinsics and the board's coordinates from diag S^-1 (fin[2 ..]: std_intrinsics).
__global__ void __launch_bounds__(256) k_ro_final(CalibRoDev d, const int* status) {
    if (*status) return;
    const CalibLM* lm = d.c.lm;
    const double sigma2 = d.c.fin[1];
    for (int a = threadIdx.x; a < d.m; a += blockDim.x) {
        const double sd = calib_ro_param_free(a, d.n, d.fixed, lm->mask) ? sqrt(d.diag[a] * sigma2) : 0.0;
        if (a < 9) d.c.fin[2 + a] = sd;
        else d.std_obj[a - 9] = sd;
    }
}

}  // namespace fid

extern "C" int fid_calibrate_camera_ro(int device, int n_views, const int32_t* offsets, const float* obj, const float* img, int width, int height,
                                       const fid_camera* guess, int32_t flags, const fid_calib_criteria* criteria, fid_calib_result* result, double* rvecs,
                                       double* tvecs, double* std_extrinsics, double* per_view_errors, fid_calib_stats* stats, int fixed_point,
                                       float* new_obj_points, double* std_obj_points, int* released) {
    using namespace fid;
    const int n = (n_views >= 1 && offsets) ? offsets[1] - offsets[0] : 0;
    if (released) *released = 0;
    if (!(fixed_point >= 1 && fixed_point <= n - 2))  // cv2 releases nothing: the standard calibration
        return fid_calibrate_camera(device, n_views, offsets, obj, img, width, height, guess, flags, criteria, result, rvecs, tvecs, std_extrinsics,
                                    per_view_errors, stats);
    if (!result) return FID_ERR_INVALID_ARG;
    memset(result, 0, sizeof(*result));
    if (stats) memset(stats, 0, sizeof(*stats));
    auto fail = [&](int why) {
        result->status = why;
        return FID_ERR_INVALID_ARG;
    };
    CalibInput ci;
    const int chk = calib_check(n_views, offsets, obj, img, width, height, guess, flags, criteria, &ci);
    if (chk < 0) return chk;
    if (chk > 0) return fail(chk);
    // cv2's collectCalibrationData with a released board: equal view sizes, then identical object points
    for (int v = 1; v < n_views; v++)
        if (offsets[v + 1] - offsets[v] != n) return fail(FID_CALIB_E_RO_VIEWS);
    for (int v = 1; v < n_views; v++)
        for (int k = 0; k < 3 * n; k++)
            if (obj[(size_t)3 * n * v + k] != obj[k]) return fail(FID_CALIB_E_RO_VIEWS);
    if (n > FID_CALIB_RO_MAX_POINTS) return fail(FID_CALIB_E_POINTS);
    if (n_views > FID_CALIB_RO_MAX_VIEWS) return fail(FID_CALIB_E_INPUT);
    {  // cv2: "There should be less vars to optimize ... than the number of residuals"
        int mask[9];
        calib_mask(flags, mask);
        if (calib_ro_nfree(mask, n_views, n) >= 2 * ci.total) return fail(FID_CALIB_E_RO_RESIDUALS);
    }
    const int total = ci.total, nv = n_views, m = 9 + 3 * n, mp = (m + DENSE_TILE - 1) / DENSE_TILE * DENSE_TILE;
    const int chunk = nv < CALIB_RO_CHUNK ? nv : CALIB_RO_CHUNK, cols = 6 * chunk;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) {
        cudaGetLastError();
        return FID_ERR_NO_DEVICE;
    }
    int prev_device = 0;
    cudaGetDevice(&prev_device);
    int rc = FID_OK, launches = 0, h_status = 0;
    cudaStream_t st = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    char* mem = nullptr;
    CalibRoDev d;
    CalibDev& c = d.c;
    std::vector<char> lm_buf(sizeof(CalibLM));
    CalibLM* h_lm = (CalibLM*)lm_buf.data();
    double init[9];
    if (ci.use_guess) {
        const double A[9] = {ci.g.K[0], ci.g.K[4], ci.g.K[2], ci.g.K[5], ci.g.D[0], ci.g.D[1], ci.g.D[2], ci.g.D[3], ci.g.D[4]};
        memcpy(init, A, sizeof(init));
    } else {
        const double A[9] = {0, 0, (width - 1) * 0.5, (height - 1) * 0.5, 0, 0, 0, 0, 0};
        memcpy(init, A, sizeof(init));
    }
    std::vector<double> board(ci.objz.begin(), ci.objz.begin() + 3 * n), h_p, h_std, h_pve, h_fin(11), h_sobj(3 * (size_t)n);
    float ms = 0.0f;
    size_t bytes = 0;
    const size_t sz_off = sizeof(int32_t) * (nv + 1), sz_obj = sizeof(float) * 3 * (size_t)total, sz_img = sizeof(float) * 2 * (size_t)total;
    auto carve = [&](size_t sz) {
        const size_t at = bytes;
        bytes += (sz + 255) & ~(size_t)255;
        return at;
    };
    const size_t o_off = carve(sz_off), o_obj = carve(sz_obj), o_img = carve(sz_img), o_mn = carve(sizeof(double) * 2 * (size_t)total),
                 o_ab = carve(sizeof(double) * 6 * nv), o_init = carve(sizeof(double) * 9), o_p = carve(sizeof(double) * 6 * nv),
                 o_pp = carve(sizeof(double) * 6 * nv), o_blk = carve(sizeof(double) * CALIB_BLK * (size_t)nv), o_trial = carve(sizeof(double) * 3 * nv),
                 o_std = carve(sizeof(double) * 6 * nv), o_pve = carve(sizeof(double) * nv), o_lm = carve(sizeof(CalibLM)), o_fin = carve(sizeof(double) * 11),
                 o_status = carve(sizeof(int)), o_board = carve(sizeof(double) * 3 * n), o_board_prev = carve(sizeof(double) * 3 * n),
                 o_pts = carve(sizeof(double) * CALIB_PT * n), o_fac = carve(sizeof(double) * CALIB_FAC * (size_t)nv), o_S = carve(sizeof(double) * (size_t)mp * mp),
                 o_r = carve(sizeof(double) * mp), o_Z = carve(sizeof(double) * (size_t)mp * cols), o_diag = carve(sizeof(double) * mp), o_on = carve(sizeof(double) * 2),
                 o_sobj = carve(sizeof(double) * 3 * n);
    const int warp_grid = (nv + 3) / 4, thread_grid = (nv + 127) / 128;
    const int max_steps = 2 * ci.max_iter + 20;
    int* d_status;
    CKC(cudaSetDevice(device));
    CKC(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    CKC(cudaEventCreate(&ev0));
    CKC(cudaEventCreate(&ev1));
    CKC(cudaMalloc(&mem, bytes));
    c.nv = nv;
    c.off = (const int32_t*)(mem + o_off);
    c.obj = (const float*)(mem + o_obj);
    c.img = (const float*)(mem + o_img);
    c.mn = (double*)(mem + o_mn);
    c.ab = (double*)(mem + o_ab);
    c.init = (double*)(mem + o_init);
    c.p = (double*)(mem + o_p);
    c.pp = (double*)(mem + o_pp);
    c.blk = (double*)(mem + o_blk);
    c.sch = nullptr;
    c.trial = (double*)(mem + o_trial);
    c.std_ext = (double*)(mem + o_std);
    c.pve = (double*)(mem + o_pve);
    c.lm = (CalibLM*)(mem + o_lm);
    c.fin = (double*)(mem + o_fin);
    d.n = n;
    d.fixed = fixed_point;
    d.m = m;
    d.mp = mp;
    d.cols = cols;
    d.board = (double*)(mem + o_board);
    d.board_prev = (double*)(mem + o_board_prev);
    d.pts = (double*)(mem + o_pts);
    d.fac = (double*)(mem + o_fac);
    d.S = (double*)(mem + o_S);
    d.r = (double*)(mem + o_r);
    d.Z = (double*)(mem + o_Z);
    d.diag = (double*)(mem + o_diag);
    d.on = (double*)(mem + o_on);
    d.std_obj = (double*)(mem + o_sobj);
    d_status = (int*)(mem + o_status);
    CKC(cudaEventRecord(ev0, st));
    CKC(cudaMemcpyAsync(mem + o_off, offsets, sz_off, cudaMemcpyHostToDevice, st));
    CKC(cudaMemcpyAsync(mem + o_obj, ci.objz.data(), sz_obj, cudaMemcpyHostToDevice, st));
    CKC(cudaMemcpyAsync(mem + o_img, img, sz_img, cudaMemcpyHostToDevice, st));
    CKC(cudaMemcpyAsync(d.board, board.data(), sizeof(double) * 3 * n, cudaMemcpyHostToDevice, st));
    CKC(cudaMemsetAsync(d_status, 0, sizeof(int), st));
    CKC(cudaMemsetAsync(d.Z, 0, sizeof(double) * (size_t)mp * cols, st));  // rows m .. mp stay 0
    CKC(cudaMemcpyAsync(c.init, init, sizeof(init), cudaMemcpyHostToDevice, st));
    if (!ci.use_guess) {
        k_calib_homography<<<warp_grid, 128, 0, st>>>(c, d_status);
        k_calib_init<<<1, 32, 0, st>>>(c, width, height, ci.aspect, d_status);
        launches += 2;
    }
    k_calib_extrinsics<<<warp_grid, 128, 0, st>>>(c, d_status);
    k_calib_lm_init<<<1, 1, 0, st>>>(c, flags, ci.aspect, ci.max_iter, ci.eps, d_status);
    launches += 2;
    {
        const int* state = &c.lm->state;
        const int point_grid = (n + 127) / 128, zgrid = (n + 128) / 128;
        const dim3 init_grid(mp / 32, mp / 8), init_block(32, 8), syrk_grid((mp + DENSE_SYRK_TILE - 1) / DENSE_SYRK_TILE, (mp + DENSE_SYRK_TILE - 1) / DENSE_SYRK_TILE);
        const size_t trsv_smem = sizeof(double) * mp;
        // the reduced system at the J's parameters (final_pass: undamped, at the final ones), factored
        auto reduce = [&](int final_pass) {
            k_ro_factor<<<thread_grid, 128, 0, st>>>(d, final_pass, d_status);
            k_ro_init<<<init_grid, init_block, 0, st>>>(d, final_pass, d_status);
            launches += 2;
            for (int v0 = 0; v0 < nv; v0 += chunk) {
                const int nvc = nv - v0 < chunk ? nv - v0 : chunk;
                k_ro_zbuild<<<dim3(zgrid, nvc), 128, 0, st>>>(d, v0, final_pass, d_status);
                if (!final_pass) k_ro_rhs<<<(mp + 127) / 128, 128, 0, st>>>(d, v0, nvc, d_status);
                k_dense_syrk<<<syrk_grid, 256, 0, st>>>(d.S, mp, mp, d.Z, 1, mp, d.Z, 1, mp, 6 * nvc, d_status, final_pass ? nullptr : state);
                launches += final_pass ? 2 : 3;
            }
            launches += dense_cholesky_enqueue(d.S, mp, FID_CALIB_E_RO_SINGULAR, d_status, final_pass ? nullptr : state, st);
        };
        for (int s = 0; s < max_steps; s++) {
            k_ro_eval<<<warp_grid, 128, 0, st>>>(d, 0, d_status);
            k_ro_points<<<point_grid, 128, 0, st>>>(d, 0, d_status);
            k_ro_sums<<<1, 64, 0, st>>>(d, 0, d_status);
            launches += 3;
            reduce(0);
            k_dense_trsv<<<1, 256, trsv_smem, st>>>(d.S, mp, mp, d.r, mp, 1, nullptr, d_status, state);
            k_ro_step<<<1, 1, 0, st>>>(d, d_status);
            k_ro_trial<<<warp_grid, 128, 0, st>>>(d, d_status);
            k_ro_decide<<<1, 32, 0, st>>>(d, d_status);
            launches += 4;
        }
        k_ro_eval<<<warp_grid, 128, 0, st>>>(d, 1, d_status);
        k_ro_points<<<point_grid, 128, 0, st>>>(d, 1, d_status);
        k_ro_sums<<<1, 64, 0, st>>>(d, 1, d_status);
        launches += 3;
        reduce(1);
        for (int v0 = 0; v0 < nv; v0 += chunk) {
            const int nvc = nv - v0 < chunk ? nv - v0 : chunk;
            k_ro_zbuild<<<dim3(zgrid, nvc), 128, 0, st>>>(d, v0, 1, d_status);
            k_dense_trsv<<<6 * nvc, 256, trsv_smem, st>>>(d.S, mp, mp, d.Z, mp, 0, nullptr, d_status, nullptr);
            k_ro_view_std<<<(nvc + 127) / 128, 128, 0, st>>>(d, v0, nvc, d_status);
            launches += 3;
        }
        for (int a0 = 0; a0 < m; a0 += cols) {
            const int ncols = m - a0 < cols ? m - a0 : cols;
            k_ro_eye<<<(int)(((size_t)ncols * mp + 255) / 256), 256, 0, st>>>(d, a0, ncols, d_status);
            k_dense_trsv<<<ncols, 256, trsv_smem, st>>>(d.S, mp, mp, d.Z, mp, 0, d.diag + a0, d_status, nullptr);
            launches += 2;
        }
        k_ro_final<<<1, 256, 0, st>>>(d, d_status);
        launches++;
    }
    CKC(cudaGetLastError());
    CKC(cudaEventRecord(ev1, st));
    h_p.resize(6 * (size_t)nv);
    h_std.resize(6 * (size_t)nv);
    h_pve.resize(nv);
    CKC(cudaMemcpyAsync(&h_status, d_status, sizeof(int), cudaMemcpyDeviceToHost, st));
    CKC(cudaMemcpyAsync(h_lm, c.lm, sizeof(CalibLM), cudaMemcpyDeviceToHost, st));
    CKC(cudaMemcpyAsync(h_p.data(), c.p, sizeof(double) * 6 * nv, cudaMemcpyDeviceToHost, st));
    CKC(cudaMemcpyAsync(h_std.data(), c.std_ext, sizeof(double) * 6 * nv, cudaMemcpyDeviceToHost, st));
    CKC(cudaMemcpyAsync(h_pve.data(), c.pve, sizeof(double) * nv, cudaMemcpyDeviceToHost, st));
    CKC(cudaMemcpyAsync(h_fin.data(), c.fin, sizeof(double) * 11, cudaMemcpyDeviceToHost, st));
    CKC(cudaMemcpyAsync(board.data(), d.board, sizeof(double) * 3 * n, cudaMemcpyDeviceToHost, st));
    CKC(cudaMemcpyAsync(h_sobj.data(), d.std_obj, sizeof(double) * 3 * n, cudaMemcpyDeviceToHost, st));
    CKC(cudaStreamSynchronize(st));
    CKC(cudaEventElapsedTime(&ms, ev0, ev1));
    if (h_status) {
        rc = fail(h_status);
        goto done;
    }
    calib_fill_result(h_lm, h_fin.data(), h_p, h_std, h_pve, nv, result, rvecs, tvecs, std_extrinsics, per_view_errors);
    if (new_obj_points)
        for (int k = 0; k < 3 * n; k++) new_obj_points[k] = (float)board[k];
    if (std_obj_points) memcpy(std_obj_points, h_sobj.data(), sizeof(double) * 3 * n);
    if (released) *released = 1;
    calib_fill_stats(h_lm, launches, ms, stats);
done:
    if (st) cudaStreamSynchronize(st);
    if (mem) cudaFree(mem);
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
    if (st) cudaStreamDestroy(st);
    cudaSetDevice(prev_device);
    return rc;
}
