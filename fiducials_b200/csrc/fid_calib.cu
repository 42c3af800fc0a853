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

extern "C" int fid_calibrate_camera(int device, int n_views, const int32_t* offsets, const float* obj, const float* img, int width, int height, const fid_camera* guess,
                                    int32_t flags, const fid_calib_criteria* criteria, fid_calib_result* result, double* rvecs, double* tvecs, double* std_extrinsics,
                                    double* per_view_errors, fid_calib_stats* stats) {
    using namespace fid;
    if (!result) return FID_ERR_INVALID_ARG;
    memset(result, 0, sizeof(*result));
    if (stats) memset(stats, 0, sizeof(*stats));
    const int supported = FID_CALIB_USE_INTRINSIC_GUESS | FID_CALIB_FIX_ASPECT_RATIO | FID_CALIB_FIX_PRINCIPAL_POINT | FID_CALIB_ZERO_TANGENT_DIST |
                          FID_CALIB_FIX_FOCAL_LENGTH | FID_CALIB_FIX_K1 | FID_CALIB_FIX_K2 | FID_CALIB_FIX_K3;
    if (flags & ~supported) return FID_ERR_UNSUPPORTED;
    auto fail = [&](int why) {
        result->status = why;
        return FID_ERR_INVALID_ARG;
    };
    if (n_views < 1 || n_views > FID_CALIB_MAX_VIEWS || !offsets || !obj || !img || width < 1 || height < 1 || offsets[0] != 0) return fail(FID_CALIB_E_INPUT);
    for (int v = 0; v < n_views; v++) {
        const int n = offsets[v + 1] - offsets[v];
        if (offsets[v + 1] < offsets[v] || offsets[v + 1] > FID_CALIB_MAX_TOTAL) return fail(FID_CALIB_E_INPUT);
        if (n < 4 || n > FID_CALIB_MAX_POINTS) return fail(FID_CALIB_E_POINTS);
    }
    const int total = offsets[n_views];
    for (size_t i = 0; i < (size_t)total * 3; i++)
        if (!std::isfinite(obj[i])) return fail(FID_CALIB_E_INPUT);
    for (size_t i = 0; i < (size_t)total * 2; i++)
        if (!std::isfinite(img[i])) return fail(FID_CALIB_E_INPUT);
    // CvLevMarq's criteria
    int max_iter = 30;
    double eps = DBL_EPSILON;
    if (criteria) {
        if (criteria->type & 1) max_iter = criteria->max_iter < 1 ? 1 : (criteria->max_iter > 1000 ? 1000 : criteria->max_iter);
        if (criteria->type & 2) {
            if (std::isnan(criteria->epsilon)) return fail(FID_CALIB_E_INPUT);
            eps = criteria->epsilon > 0 ? criteria->epsilon : 0.0;
        }
    }
    fid_camera g;
    memset(&g, 0, sizeof(g));
    g.K[0] = g.K[4] = g.K[8] = 1.0;
    if (guess) g = *guess;
    else if (flags & FID_CALIB_USE_INTRINSIC_GUESS) return fail(FID_CALIB_E_GUESS);
    for (int k = 0; k < 9; k++)
        if (!std::isfinite(g.K[k]) || (k < 5 && !std::isfinite(g.D[k]))) return fail(FID_CALIB_E_INPUT);
    const bool use_guess = flags & FID_CALIB_USE_INTRINSIC_GUESS;
    if (use_guess) {
        const double* K = g.K;
        if (K[0] <= 0 || K[4] <= 0 || K[2] < 0 || K[2] >= width || K[5] < 0 || K[5] >= height || fabs(K[1]) > 1e-5 || fabs(K[3]) > 1e-5 || fabs(K[6]) > 1e-5 ||
            fabs(K[7]) > 1e-5 || fabs(K[8] - 1) > 1e-5)
            return fail(FID_CALIB_E_GUESS);
    }
    double aspect = 0.0;
    if (flags & FID_CALIB_FIX_ASPECT_RATIO) {
        aspect = g.K[0] / g.K[4];
        if (!(aspect >= 0.01 && aspect <= 100.0)) return fail(FID_CALIB_E_GUESS);
    }
    std::vector<float> objz(obj, obj + (size_t)total * 3);
    if (!use_guess) {  // planar rigs only: meanStdDev of z, then z = 0
        double s = 0.0, sq = 0.0;
        for (int i = 0; i < total; i++) {
            const double z = obj[3 * i + 2];
            s += z;
            sq += z * z;
        }
        const double mean = s / total, var = sq / total - mean * mean, sdv = sqrt(var > 0 ? var : 0.0);
        if (fabs(mean) > 1e-5 || sdv > 1e-5) return fail(FID_CALIB_E_NONPLANAR);
        for (int i = 0; i < total; i++) objz[3 * i + 2] = 0.0f;
    }
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
    result->rms = h_fin[0];
    memset(&result->camera, 0, sizeof(result->camera));
    result->camera.K[0] = h_lm->in[0];
    result->camera.K[2] = h_lm->in[2];
    result->camera.K[4] = h_lm->in[1];
    result->camera.K[5] = h_lm->in[3];
    result->camera.K[8] = 1.0;
    for (int k = 0; k < 5; k++) result->camera.D[k] = h_lm->in[4 + k];
    for (int a = 0; a < 9; a++) result->std_intrinsics[a] = h_fin[2 + a];
    result->iterations = h_lm->iters;
    for (int v = 0; v < nv; v++)
        for (int k = 0; k < 3; k++) {
            if (rvecs) rvecs[3 * v + k] = h_p[6 * v + k];
            if (tvecs) tvecs[3 * v + k] = h_p[6 * v + 3 + k];
        }
    if (std_extrinsics) memcpy(std_extrinsics, h_std.data(), sizeof(double) * 6 * nv);
    if (per_view_errors) memcpy(per_view_errors, h_pve.data(), sizeof(double) * nv);
    if (stats) {
        stats->n_steps = h_lm->n_steps;
        stats->n_evaluations = h_lm->n_evals;
        stats->kernel_launches = launches;
        stats->device_ms = ms;
        memcpy(stats->steps, h_lm->steps, h_lm->n_steps < FID_CALIB_MAX_STEPS ? h_lm->n_steps : FID_CALIB_MAX_STEPS);
    }
done:
    if (st) cudaStreamSynchronize(st);
    if (mem) cudaFree(mem);
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
    if (st) cudaStreamDestroy(st);
    cudaSetDevice(prev_device);
    return rc;
}
