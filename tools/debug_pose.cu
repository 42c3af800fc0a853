// Debug aid: run solve_marker_pose on host and device from the same translation unit and print the
// LM trajectory of both.  nvcc -gencode arch=compute_90a,code=sm_90a --fmad=false -DFID_DEBUG_PNP tools/debug_pose.cu
#include <cstdio>
#include <cuda_runtime.h>
#include "../fiducials_b200/csrc/pnp.cuh"
using namespace fid;
__global__ void k(const float* c, Camera cam, PoseOut* out) { solve_marker_pose(c, cam, 0.14f, 0.14, out); }
int main() {
    // C1 seed 0 marker 0 corners (from the oracle) and camera
    float c[8] = {174.0747f, 105.04338f, 129.32097f, 208.1023f, 13.963207f, 167.47575f, 67.718f, 60.5f};  // any 4 marker corners
    Camera cam = {0.73 * 640, 0.73 * 640, 320, 240, 0.1349735087283542, -0.2335869827451621, 0.0006697030315075139, 0.004846737465872353, 0.0};
    PoseOut h;
    printf("--- host\n");
    solve_marker_pose(c, cam, 0.14f, 0.14, &h);
    printf("host rvec %.9f %.9f %.9f iters %d\n", h.rvec[0], h.rvec[1], h.rvec[2], h.lm_iters);
    float* dc; PoseOut* dout;
    cudaMalloc(&dc, sizeof(c)); cudaMalloc(&dout, sizeof(PoseOut));
    cudaMemcpy(dc, c, sizeof(c), cudaMemcpyHostToDevice);
    printf("--- device\n");
    k<<<1, 1>>>(dc, cam, dout);
    cudaDeviceSynchronize();
    PoseOut d;
    cudaMemcpy(&d, dout, sizeof(d), cudaMemcpyDeviceToHost);
    printf("dev  rvec %.9f %.9f %.9f iters %d\n", d.rvec[0], d.rvec[1], d.rvec[2], d.lm_iters);
    return 0;
}
