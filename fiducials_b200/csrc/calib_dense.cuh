// Dense FP64 kernels of the reduced systems of fid_calibrate_camera_ro (calib.cuh, "object release") and fid_map_bundle_adjust
// (map_ba.cuh), for sm_90a.
//
// Matrices are row-major with a leading dimension `ld` that is a multiple of 32 (the padded size mp >= m); only the lower
// triangle of the symmetric system is computed and read.  Every kernel sums in a fixed order and uses no atomics, so two runs
// give the same bits.  Every kernel returns at once when *status is set or the run is done (*state == 2; state may be null).
//   k_dense_syrk   C(lower tiles) -= A B^T over k, 64x64 tiles per 256-thread CTA on mma.sync.m8n8k4.f64 (a warp: 16x32)
//   k_dense_potrf  one CTA: Cholesky of the 32x32 diagonal block at (j0, j0); a non-positive pivot sets *status
//   k_dense_trsm   thread per row below it: the panel L21 = A21 L11^-T
//   k_dense_trsv   CTA per right-hand side (a column of length ld): L y = x, then (backward) L^T x = y, blocked by 32
// A blocked right-looking factorisation is potrf / trsm / syrk per 32-column panel (dense_cholesky_enqueue).
// The kernels are static: every translation unit that includes this file (fid_calib.cu, fid_map_ba.cu) gets its own copy.
#pragma once
#include <cuda_runtime.h>

namespace fid {

#define DENSE_TILE 32
#define DENSE_KC 16
#define DENSE_SYRK_TILE 64

__device__ __forceinline__ void dense_mma(double a, double b, double& c0, double& c1) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};\n" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

__device__ __forceinline__ bool dense_stop(const int* status, const int* state) { return *(volatile const int*)status != 0 || (state && *(volatile const int*)state == 2); }

// C[i][j] -= sum_k A(i, k) B(j, k) for the 64x64 tiles with tile row >= tile column of the n x n block C (ldc), n a multiple of
// 32; A(i, k) = A[i * sai + k * sak], B(j, k) likewise.  Grid (ceil(n / 64), ceil(n / 64)) of 256 threads; the upper tiles return
// at once.  A warp computes 16x32 of the tile as 2x4 mma.m8n8k4 tiles, K in steps of 16 staged in shared memory.
static __global__ void __launch_bounds__(256) k_dense_syrk(double* C, int ldc, int n, const double* A, size_t sai, size_t sak, const double* B, size_t sbj,
                                                    size_t sbk, int K, const int* status, const int* state) {
    const int ti = blockIdx.y, tj = blockIdx.x;
    if (tj > ti || dense_stop(status, state)) return;
    __shared__ double As[DENSE_SYRK_TILE][DENSE_KC + 1], Bs[DENSE_SYRK_TILE][DENSE_KC + 1];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wr = (warp >> 1) * 16, wc = (warp & 1) * 32;  // the warp's 16x32 part
    const int i0 = ti * DENSE_SYRK_TILE, j0 = tj * DENSE_SYRK_TILE;
    double acc[2][4][2] = {};
    for (int k0 = 0; k0 < K; k0 += DENSE_KC) {
        for (int e = threadIdx.x; e < DENSE_SYRK_TILE * DENSE_KC; e += 256) {
            // consecutive threads along the tile rows or along k, whichever is contiguous in memory
            const int r = sai == 1 ? e % DENSE_SYRK_TILE : e / DENSE_KC, kk = sai == 1 ? e / DENSE_SYRK_TILE : e % DENSE_KC;
            const bool in = k0 + kk < K;
            As[r][kk] = in && i0 + r < n ? A[(size_t)(i0 + r) * sai + (size_t)(k0 + kk) * sak] : 0.0;
            Bs[r][kk] = in && j0 + r < n ? B[(size_t)(j0 + r) * sbj + (size_t)(k0 + kk) * sbk] : 0.0;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < DENSE_KC; kk += 4) {
            double a[2], b[4];
#pragma unroll
            for (int x = 0; x < 2; x++) a[x] = As[wr + 8 * x + (lane >> 2)][kk + (lane & 3)];
#pragma unroll
            for (int y = 0; y < 4; y++) b[y] = Bs[wc + 8 * y + (lane >> 2)][kk + (lane & 3)];
#pragma unroll
            for (int x = 0; x < 2; x++)
#pragma unroll
                for (int y = 0; y < 4; y++) dense_mma(a[x], b[y], acc[x][y][0], acc[x][y][1]);
        }
        __syncthreads();
    }
    const int r = i0 + wr + (lane >> 2);
#pragma unroll
    for (int x = 0; x < 2; x++)
#pragma unroll
        for (int y = 0; y < 4; y++) {
            const int c = j0 + wc + 8 * y + 2 * (lane & 3);
            if (r + 8 * x >= n || c >= n) continue;  // n is a multiple of 32: a pair of columns is inside or outside together
            double* p = C + (size_t)(r + 8 * x) * ldc + c;
            p[0] -= acc[x][y][0];
            p[1] -= acc[x][y][1];
        }
}

// One CTA of 32 x 32 threads: the Cholesky factor of the diagonal block at (j0, j0), in place (lower).
static __global__ void __launch_bounds__(1024) k_dense_potrf(double* S, int ld, int j0, int fail_status, int* status, const int* state) {
    if (dense_stop(status, state)) return;
    __shared__ double a[DENSE_TILE][DENSE_TILE + 1];
    __shared__ int bad;
    const int r = threadIdx.y, c = threadIdx.x;
    a[r][c] = S[(size_t)(j0 + r) * ld + j0 + c];
    if (r == 0 && c == 0) bad = 0;
    __syncthreads();
    for (int k = 0; k < DENSE_TILE; k++) {
        if (r == k && c == k) {
            if (!(a[k][k] > 0.0)) bad = 1;
            a[k][k] = sqrt(a[k][k] > 0.0 ? a[k][k] : 1.0);
        }
        __syncthreads();
        if (c == k && r > k) a[r][k] /= a[k][k];
        __syncthreads();
        if (r > k && c > k && c <= r) a[r][c] -= a[r][k] * a[c][k];
        __syncthreads();
    }
    if (c <= r) S[(size_t)(j0 + r) * ld + j0 + c] = a[r][c];
    if (r == 0 && c == 0 && bad) *status = fail_status;
}

// Thread per row i >= j0 + 32 (below the diagonal block, up to n): L[i][j0..j0+32) = A[i][j0..j0+32) L11^-T.
static __global__ void __launch_bounds__(128) k_dense_trsm(double* S, int ld, int j0, int n, const int* status, const int* state) {
    if (dense_stop(status, state)) return;
    __shared__ double l[DENSE_TILE][DENSE_TILE + 1];
    for (int e = threadIdx.x; e < DENSE_TILE * DENSE_TILE; e += blockDim.x) l[e / DENSE_TILE][e % DENSE_TILE] = S[(size_t)(j0 + e / DENSE_TILE) * ld + j0 + e % DENSE_TILE];
    __syncthreads();
    const int i = j0 + DENSE_TILE + blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double* row = S + (size_t)i * ld + j0;
    double x[DENSE_TILE];
#pragma unroll
    for (int c = 0; c < DENSE_TILE; c++) {
        double s = row[c];
#pragma unroll
        for (int k = 0; k < c; k++) s -= x[k] * l[c][k];
        x[c] = s / l[c][c];
    }
#pragma unroll
    for (int c = 0; c < DENSE_TILE; c++) row[c] = x[c];
}

// CTA per right-hand side X + b * ldx (n = the padded size, a multiple of 32): L y = x and, with `backward`, L^T x = y, in place.
// With norms != null, norms[b] = |y|^2 (summed in row order) after the forward solve.
static __global__ void __launch_bounds__(256) k_dense_trsv(const double* L, int ld, int n, double* X, size_t ldx, int backward, double* norms, const int* status,
                                                    const int* state) {
    if (dense_stop(status, state)) return;
    extern __shared__ double x[];
    double* xg = X + ldx * blockIdx.x;
    for (int i = threadIdx.x; i < n; i += blockDim.x) x[i] = xg[i];
    __syncthreads();
    for (int b = 0; b < n; b += DENSE_TILE) {
        if (threadIdx.x < 32) {  // the diagonal block: lane r holds row b + r and finalises x[b + r]
            const int lane = threadIdx.x;
            double l[DENSE_TILE], xi = x[b + lane];
#pragma unroll
            for (int k = 0; k < DENSE_TILE; k++) l[k] = L[(size_t)(b + lane) * ld + b + k];
#pragma unroll
            for (int i = 0; i < DENSE_TILE; i++) {
                if (lane == i) xi /= l[i];
                const double xv = __shfl_sync(0xffffffffu, xi, i);
                if (lane > i) xi -= l[i] * xv;
            }
            x[b + lane] = xi;
        }
        __syncthreads();
        for (int i = b + DENSE_TILE + threadIdx.x; i < n; i += blockDim.x) {
            double s = x[i];
            for (int k = b; k < b + DENSE_TILE; k++) s -= L[(size_t)i * ld + k] * x[k];
            x[i] = s;
        }
        __syncthreads();
    }
    if (norms && threadIdx.x == 0) {
        double s = 0.0;
        for (int i = 0; i < n; i++) s += x[i] * x[i];
        norms[blockIdx.x] = s;
    }
    if (backward)
        for (int b = n - DENSE_TILE; b >= 0; b -= DENSE_TILE) {
            if (threadIdx.x < 32) {  // lane r holds column b + r of the block
                const int lane = threadIdx.x;
                double l[DENSE_TILE], xi = x[b + lane];
#pragma unroll
                for (int k = 0; k < DENSE_TILE; k++) l[k] = L[(size_t)(b + k) * ld + b + lane];
#pragma unroll
                for (int i = DENSE_TILE - 1; i >= 0; i--) {
                    if (lane == i) xi /= l[i];
                    const double xv = __shfl_sync(0xffffffffu, xi, i);
                    if (lane < i) xi -= l[i] * xv;
                }
                x[b + lane] = xi;
            }
            __syncthreads();
            for (int i = threadIdx.x; i < b; i += blockDim.x) {
                double s = x[i];
                for (int k = b; k < b + DENSE_TILE; k++) s -= L[(size_t)k * ld + i] * x[k];
                x[i] = s;
            }
            __syncthreads();
        }
    for (int i = threadIdx.x; i < n; i += blockDim.x) xg[i] = x[i];
}

// Enqueue the blocked right-looking Cholesky of the n x n lower triangle of S (n a multiple of 32): 3 launches per panel.
static inline int dense_cholesky_enqueue(double* S, int n, int fail_status, int* status, const int* state, cudaStream_t st) {
    int launches = 0;
    for (int j0 = 0; j0 < n; j0 += DENSE_TILE) {
        k_dense_potrf<<<1, dim3(DENSE_TILE, DENSE_TILE), 0, st>>>(S, n, j0, fail_status, status, state);
        launches++;
        const int rest = n - j0 - DENSE_TILE;
        if (rest == 0) break;
        k_dense_trsm<<<(rest + 127) / 128, 128, 0, st>>>(S, n, j0, n, status, state);
        double* P = S + (size_t)(j0 + DENSE_TILE) * n + j0;
        const int g = (rest + DENSE_SYRK_TILE - 1) / DENSE_SYRK_TILE;
        k_dense_syrk<<<dim3(g, g), 256, 0, st>>>(P + DENSE_TILE, n, rest, P, n, 1, P, n, 1, DENSE_TILE, status, state);
        launches += 2;
    }
    return launches;
}

}  // namespace fid
