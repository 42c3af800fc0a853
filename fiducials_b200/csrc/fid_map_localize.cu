// fid_map_localize: one camera pose per frame from every visible mapped marker's corners, with its covariance (map_localize.cuh
// states the computation, DESIGN.md f17).
//
// k_map_localize runs a warp per frame.  The lanes look the frame's ids up in the instance (through its id -> slot hash when that
// is valid, linearly otherwise: fid_map_load and a merge leave it stale until the next fold rebuilds it), test the duplicates,
// and stage the counted markers' float32 board in the frame's scratch, compacted in detection order by a ballot prefix; then all
// 32 lanes run loc_solve together (board_sum's lane model: fixed summation orders, no atomics) and lane 0 writes the record.
// Everything runs on the map's stream, so the kernel sees the map as pending asynchronous updates leave it.
#include "map_localize.cuh"

#include <cuda_runtime.h>
#include <math.h>
#include <string.h>

#include <algorithm>

#include "fid_map_internal.h"

namespace fid {

struct LocArgs {
    int n_frames, mm, ms;  // frames, the layout's max_markers, scratch markers per frame
    const int32_t *counts, *ids;
    const float* corners;
    const MapState* state;
    const MapEntry* entries;
    MapHash hash;
    Camera cam;
    double fiducial_len, max_entry_variance;
    int n_override;
    const int32_t* override_ids;
    const double* override_lens;
    int have_base;
    Twv camBase;
    float *obj, *img, *len_f;  // [F][4 ms][3], [F][4 ms][2], [F][ms]
    double *mn, *mpose;        // [F][4 ms][2], [F][ms][12]
    fid_localization* out;
};

__global__ void __launch_bounds__(128) k_map_localize(const LocArgs a) {
    const int f = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (f >= a.n_frames) return;
    const MapState st = *a.state;
    const MapHash* h = st.hash_valid && a.hash.size > 0 ? &a.hash : nullptr;
    const int n = a.counts[f];
    const int32_t* fid = a.ids + (size_t)f * a.mm;
    const float* fc = a.corners + (size_t)f * a.mm * 8;
    float* obj = a.obj + (size_t)f * a.ms * 12;
    float* img = a.img + (size_t)f * a.ms * 8;
    float* len_f = a.len_f + (size_t)f * a.ms;
    double* mn = a.mn + (size_t)f * a.ms * 8;
    double* mpose = a.mpose + (size_t)f * a.ms * 12;
    int used = 0;
    for (int j0 = 0; j0 < n; j0 += 32) {
        const int j = j0 + lane;
        const int s = j < n ? loc_slot(st, a.entries, h, n, fid, j, a.max_entry_variance) : -1;
        const unsigned mask = __ballot_sync(0xffffffffu, s >= 0);
        if (s >= 0) {
            const int k = used + __popc(mask & ((1u << lane) - 1u));
            loc_stage_marker(a.entries[s], ba_marker_len(fid[j], a.fiducial_len, a.n_override, a.override_ids, a.override_lens), fc + 8 * (size_t)j, obj + 12 * k,
                             img + 8 * k, len_f + k, mpose + 12 * k);
        }
        used += __popc(mask);
    }
    __syncwarp();
    fid_localization r;
    loc_solve(used, obj, img, mn, a.cam, len_f, mpose, a.fiducial_len, a.have_base ? &a.camBase : nullptr, &r);
    if (lane == 0) memcpy(a.out + f, &r, sizeof(r));  // every byte, padding included
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

extern "C" int fid_map_localize(fid_map* m, int instance, int n_frames, const int32_t* counts, const int32_t* ids, const float* corners, int max_markers,
                                const fid_camera* cam, double fiducial_len, int n_override, const int32_t* override_ids, const double* override_lens,
                                double max_entry_variance, const fid_tf* T_camBase, fid_localization* out) {
    using namespace fid;
    if (!m || instance < 0 || instance >= m->p.n_instances || n_frames < 1 || !counts || !ids || !corners || !out || max_markers < 1 ||
        max_markers > FID_MAX_MARKERS || !cam || !finite_camera(cam) || !(fiducial_len > 0) || !std::isfinite(fiducial_len) || n_override < 0 ||
        (n_override > 0 && (!override_ids || !override_lens)) || std::isnan(max_entry_variance))
        return FID_ERR_INVALID_ARG;
    for (int k = 0; k < n_override; k++)
        if (!(override_lens[k] > 0) || !std::isfinite(override_lens[k])) return FID_ERR_INVALID_ARG;
    Twv camBase{};
    if (T_camBase) {
        double qn = 0.0;
        for (int k = 0; k < 4; k++) qn += T_camBase->q[k] * T_camBase->q[k];
        for (int k = 0; k < 3; k++)
            if (!std::isfinite(T_camBase->t[k])) return FID_ERR_INVALID_ARG;
        if (!(qn > 0) || !std::isfinite(qn)) return FID_ERR_INVALID_ARG;
        q_to_m(T_camBase->q, camBase.R);
        for (int k = 0; k < 3; k++) camBase.t[k] = T_camBase->t[k];
    }
    if (n_frames > BA_MAX_FRAMES) return FID_ERR_CAPACITY;
    int ms = 1;
    for (int f = 0; f < n_frames; f++) {
        if (counts[f] < 0 || counts[f] > max_markers) return FID_ERR_INVALID_ARG;
        const float* c = corners + (size_t)8 * max_markers * f;
        for (int k = 0; k < 8 * counts[f]; k++)
            if (!std::isfinite(c[k])) return FID_ERR_INVALID_ARG;
        ms = std::max(ms, counts[f]);
    }
    const size_t F = (size_t)n_frames, cells = F * max_markers;
    size_t bytes = 0;
    auto carve = [&](size_t sz) {
        const size_t at = bytes;
        bytes += (sz + 255) & ~(size_t)255;
        return at;
    };
    const size_t a_counts = carve(sizeof(int32_t) * F), a_ids = carve(sizeof(int32_t) * cells), a_corners = carve(sizeof(float) * 8 * cells),
                 a_ovi = carve(sizeof(int32_t) * std::max(n_override, 1)), a_ovl = carve(sizeof(double) * std::max(n_override, 1)),
                 a_obj = carve(sizeof(float) * 12 * F * ms), a_img = carve(sizeof(float) * 8 * F * ms), a_len = carve(sizeof(float) * F * ms),
                 a_mn = carve(sizeof(double) * 8 * F * ms), a_mpose = carve(sizeof(double) * 12 * F * ms), a_out = carve(sizeof(fid_localization) * F);
    CK(cudaSetDevice(m->device));
    cudaStream_t st = m->stream;
    if (bytes > m->loc_cap) {
        CK(cudaStreamSynchronize(st));
        if (m->d_loc) CK(cudaFree(m->d_loc));
        m->d_loc = nullptr;
        m->loc_cap = 0;
        CK(cudaMalloc((void**)&m->d_loc, bytes));
        m->loc_cap = bytes;
    }
    char* mem = m->d_loc;
    CK(cudaMemcpyAsync(mem + a_counts, counts, sizeof(int32_t) * F, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(mem + a_ids, ids, sizeof(int32_t) * cells, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(mem + a_corners, corners, sizeof(float) * 8 * cells, cudaMemcpyHostToDevice, st));
    if (n_override) {
        CK(cudaMemcpyAsync(mem + a_ovi, override_ids, sizeof(int32_t) * n_override, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(mem + a_ovl, override_lens, sizeof(double) * n_override, cudaMemcpyHostToDevice, st));
    }
    const int cap = m->p.max_fiducials;
    LocArgs a;
    a.n_frames = n_frames;
    a.mm = max_markers;
    a.ms = ms;
    a.counts = (const int32_t*)(mem + a_counts);
    a.ids = (const int32_t*)(mem + a_ids);
    a.corners = (const float*)(mem + a_corners);
    a.state = m->d_state + instance;
    a.entries = m->d_entries + (size_t)instance * cap;
    a.hash = MapHash{m->d_hash + (size_t)instance * 2 * m->hash_size, m->d_hash + (size_t)instance * 2 * m->hash_size + m->hash_size, m->hash_size};
    a.cam = Camera{cam->K[0], cam->K[4], cam->K[2], cam->K[5], cam->D[0], cam->D[1], cam->D[2], cam->D[3], cam->D[4]};
    a.fiducial_len = fiducial_len;
    a.max_entry_variance = max_entry_variance;
    a.n_override = n_override;
    a.override_ids = (const int32_t*)(mem + a_ovi);
    a.override_lens = (const double*)(mem + a_ovl);
    a.have_base = T_camBase != nullptr;
    a.camBase = camBase;
    a.obj = (float*)(mem + a_obj);
    a.img = (float*)(mem + a_img);
    a.len_f = (float*)(mem + a_len);
    a.mn = (double*)(mem + a_mn);
    a.mpose = (double*)(mem + a_mpose);
    a.out = (fid_localization*)(mem + a_out);
    k_map_localize<<<(n_frames + 3) / 4, 128, 0, st>>>(a);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(out, a.out, sizeof(fid_localization) * F, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return FID_OK;
}
