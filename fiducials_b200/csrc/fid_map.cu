// C-ABI of the fiducial_slam map update (include/fiducials_b200.h, "Map" section).
// One CUDA thread per map instance runs the reference's sequential fold (slam.cuh); a whole
// sequence of messages can be replayed in a single launch.  The merge step for multi-GPU runs is
// new (SURVEY.md 8e) and deterministic: tables are folded in rank order, ids ascending.
#include <cuda_runtime.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../include/fiducials_b200.h"
#include "slam.cuh"

using namespace fid;



#include "fid_map_internal.h"

struct SeqArgs {
    MapState* state;
    MapEntry* entries;
    uint32_t* links;
    int cap, links_wpr;
    int32_t* hash;
    int hash_size;
    int n_instances, n_msgs;
    const int32_t* offsets;  // [n_instances][n_msgs+1]
    const Obs* obs;
    double* var_scratch;
    int* slot_scratch;
    const Twv* tf;  // [0] baseCam [1] camBase
    int have_base_cam, have_cam_base;
    double weighting_scale, systematic_error;
    int use_area;
    RobotPose* robot;  // [n_instances][n_msgs] or null
};

__global__ void k_map_sequence(const SeqArgs a) {
    const int inst = blockIdx.x * blockDim.x + threadIdx.x;
    if (inst >= a.n_instances) return;
    MapState st = a.state[inst];
    MapEntry* e = a.entries + (size_t)inst * a.cap;
    uint32_t* links = a.links ? a.links + (size_t)inst * a.cap * a.links_wpr : nullptr;
    const int32_t* off = a.offsets + (size_t)inst * (a.n_msgs + 1);
    MapHash hash{a.hash + (size_t)inst * 2 * a.hash_size, a.hash + (size_t)inst * 2 * a.hash_size + a.hash_size, a.hash_size};
    for (int k = 0; k < a.n_msgs; k++) {
        RobotPose rp;
        map_update(st, e, links, a.obs + off[k], off[k + 1] - off[k], a.have_base_cam ? &a.tf[0] : nullptr, a.have_cam_base ? &a.tf[1] : nullptr, a.weighting_scale,
                   a.use_area, a.systematic_error, &rp, &hash, a.var_scratch + off[k], a.slot_scratch + off[k]);
        if (a.robot) a.robot[(size_t)inst * a.n_msgs + k] = rp;
    }
    a.state[inst] = st;
}

// export: slot i of the table = i-th fiducial in ascending id order; unused slots id = -1
__global__ void k_map_export(const MapState* state, const MapEntry* entries, int cap, int inst, fid_map_record* table) {
    const MapState st = state[inst];
    const MapEntry* e = entries + (size_t)inst * cap;
    for (int i = threadIdx.x; i < cap; i += blockDim.x) {
        fid_map_record r;
        r.fiducial_id = -1;
        r.num_obs = 0;
        r.t[0] = r.t[1] = r.t[2] = 0;
        r.q[0] = r.q[1] = r.q[2] = 0;
        r.q[3] = 1;
        r.variance = 0;
        if (i < st.n) {
            int rank = 0;
            for (int j = 0; j < st.n; j++) rank += e[j].id < e[i].id ? 1 : 0;
            r.fiducial_id = e[i].id;
            r.num_obs = e[i].num_obs;
            r.t[0] = e[i].pose.t[0];
            r.t[1] = e[i].pose.t[1];
            r.t[2] = e[i].pose.t[2];
            m_to_q(e[i].pose.R, r.q);
            r.variance = e[i].pose.var;
            table[rank] = r;
        }
        if (i >= st.n) table[i] = r;
    }
}

// ---- merged view (multi-GPU, SURVEY 8e; no reference counterpart) --------------------------------------
// The per-rank LOCAL maps are never written by a merge: the gathered tables are folded into a separate
// "merged view" that is rebuilt from scratch by every merge, so merging the same tables twice gives the
// same view (idempotent) and information exchanged at epoch k is not fused again at epoch k+1.
// Tables are id-ascending with the unused records (-1) at the end (k_map_export).  One thread per
// (table, record): the record of the LOWEST rank that holds an id owns it and folds the higher ranks in
// rank order (TransformWithVariance::update, variance-0 entries win) -- the same order as
// oracle/slam_oracle.py::merge_maps.  Owners are then ranked by id (bitonic sort in shared memory).
#define MERGE_MAX_KEYS 4096
__device__ __forceinline__ int merge_key(int id) { return id < 0 ? 0x7fffffff : id; }
__device__ int table_find(const fid_map_record* tab, int cap, int id) {
    int lo = 0, hi = cap;  // first record with key >= id
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (merge_key(tab[mid].fiducial_id) < id)
            lo = mid + 1;
        else
            hi = mid;
    }
    return (lo < cap && tab[lo].fiducial_id == id) ? lo : -1;
}
__device__ void merge_fold(const fid_map_record* tables, int cap, int n_tables, int t0, int i0, MapEntry* out) {
    const fid_map_record& r0 = tables[(size_t)t0 * cap + i0];
    Twv pose;
    q_to_m(r0.q, pose.R);
    pose.t[0] = r0.t[0];
    pose.t[1] = r0.t[1];
    pose.t[2] = r0.t[2];
    pose.var = r0.variance;
    int num = r0.num_obs;
    for (int t = t0 + 1; t < n_tables; t++) {
        const fid_map_record* tab = tables + (size_t)t * cap;
        const int j = table_find(tab, cap, r0.fiducial_id);
        if (j < 0) continue;
        num += tab[j].num_obs;
        if (pose.var == 0.0) continue;  // pinned entry wins
        Twv other;
        q_to_m(tab[j].q, other.R);
        other.t[0] = tab[j].t[0];
        other.t[1] = tab[j].t[1];
        other.t[2] = tab[j].t[2];
        other.var = tab[j].variance;
        if (other.var == 0.0)
            pose = other;
        else
            twv_update(pose, other);
    }
    out->id = r0.fiducial_id;
    out->num_obs = num;
    out->pose = pose;
}

struct MergedHeader {
    int32_t n;
    int32_t overflow;
};

__global__ void __launch_bounds__(1024) k_map_merge_view(int cap, int n_tables, const fid_map_record* tables, MapEntry* merged, MergedHeader* hdr) {
    __shared__ unsigned long long keys[MERGE_MAX_KEYS];
    const int total = n_tables * cap;
    for (int e = threadIdx.x; e < MERGE_MAX_KEYS; e += blockDim.x) {
        unsigned long long k = ~0ull;
        if (e < total) {
            const int t = e / cap, i = e - t * cap;
            const int id = tables[e].fiducial_id;
            bool owner = id >= 0;
            for (int t2 = 0; owner && t2 < t; t2++) owner = table_find(tables + (size_t)t2 * cap, cap, id) < 0;
            if (owner) k = ((unsigned long long)(unsigned int)id << 32) | (unsigned int)e;
            (void)i;
        }
        keys[e] = k;
    }
    __syncthreads();
    for (int k = 2; k <= MERGE_MAX_KEYS; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int e = threadIdx.x; e < MERGE_MAX_KEYS; e += blockDim.x) {
                const int p = e ^ j;
                if (p > e) {
                    const unsigned long long a = keys[e], b = keys[p];
                    const bool up = (e & k) == 0;
                    if ((a > b) == up) {
                        keys[e] = b;
                        keys[p] = a;
                    }
                }
            }
            __syncthreads();
        }
    for (int e = threadIdx.x; e < MERGE_MAX_KEYS; e += blockDim.x) {
        const unsigned long long k = keys[e];
        const bool valid = k != ~0ull;
        if (valid && e < cap) {
            const int src = (int)(unsigned int)k;
            merge_fold(tables, cap, n_tables, src / cap, src % cap, &merged[e]);
        }
        const bool last = valid && (e + 1 == MERGE_MAX_KEYS || keys[e + 1] == ~0ull);
        if (last) {
            hdr->n = e + 1 < cap ? e + 1 : cap;
            hdr->overflow = e + 1 > cap ? 1 : 0;
        }
        if (e == 0 && !valid) {
            hdr->n = 0;
            hdr->overflow = 0;
        }
    }
}

// More than MERGE_MAX_KEYS records in all tables together: one thread does the k-way merge (rare; the
// tables of 8 ranks x 512 fiducials fit the parallel kernel).
__global__ void k_map_merge_view_serial(int cap, int n_tables, const fid_map_record* tables, MapEntry* merged, MergedHeader* hdr) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    int n = 0, overflow = 0;
    int last_id = -1;
    for (;;) {
        int best = 0x7fffffff, bt = -1, bi = -1;  // smallest id > last_id, lowest rank first
        for (int t = 0; t < n_tables; t++) {
            const fid_map_record* tab = tables + (size_t)t * cap;
            int lo = 0, hi = cap;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (merge_key(tab[mid].fiducial_id) <= last_id)
                    lo = mid + 1;
                else
                    hi = mid;
            }
            if (lo < cap && tab[lo].fiducial_id >= 0 && tab[lo].fiducial_id < best) {
                best = tab[lo].fiducial_id;
                bt = t;
                bi = lo;
            }
        }
        if (bt < 0) break;
        if (n < cap)
            merge_fold(tables, cap, n_tables, bt, bi, &merged[n++]);
        else
            overflow = 1;
        last_id = best;
    }
    hdr->n = n;
    hdr->overflow = overflow;
}

// adopt: the merged view replaces an instance's content (explicit; e.g. a localisation-only map at the end of a run)
__global__ void k_map_adopt(MapState* state, MapEntry* entries, uint32_t* links, int cap, int links_wpr, int inst, const MapEntry* merged, const MergedHeader* hdr) {
    MapEntry* e = entries + (size_t)inst * cap;
    const int n = hdr->n;
    for (int i = threadIdx.x; i < n; i += blockDim.x) e[i] = merged[i];
    for (int i = threadIdx.x; i < cap * links_wpr; i += blockDim.x) links[(size_t)inst * cap * links_wpr + i] = 0;  // links are per-rank bookkeeping (slot indexed)
    if (threadIdx.x == 0) {
        MapState st = state[inst];
        st.n = n;
        st.hash_valid = 0;
        if (hdr->overflow) st.overflow = 1;
        state[inst] = st;
    }
}

extern "C" int fid_map_default_params(fid_map_params* p) {
    if (!p) return FID_ERR_INVALID_ARG;
    p->weighting_scale = 1e9;
    p->use_fiducial_area_as_weight = 0;
    p->read_only_map = 0;
    p->systematic_error = 0.01;
    p->max_fiducials = 512;
    p->n_instances = 1;
    return FID_OK;
}

static int reset_state(fid_map* m, int inst_lo, int inst_hi) {
    std::vector<MapState> st(inst_hi - inst_lo);
    for (auto& s : st) {
        memset(&s, 0, sizeof(s));
        s.capacity = m->p.max_fiducials;
        s.origin_fid = -1;
        s.fiducial_to_add = -1;
        s.read_only = m->p.read_only_map;
        s.hash_size = m->hash_size;
        s.hash_valid = 0;
    }
    CK(cudaMemcpy(m->d_state + inst_lo, st.data(), sizeof(MapState) * st.size(), cudaMemcpyHostToDevice));
    const size_t wpr = (m->p.max_fiducials + 31) / 32;
    CK(cudaMemset(m->d_links + (size_t)inst_lo * m->p.max_fiducials * wpr, 0, sizeof(uint32_t) * (size_t)(inst_hi - inst_lo) * m->p.max_fiducials * wpr));
    return FID_OK;
}

extern "C" int fid_map_create(const fid_map_params* p, int device, fid_map** out) {
    if (!p || !out || p->max_fiducials < 1 || p->max_fiducials > 65536 || p->n_instances < 1) return FID_ERR_INVALID_ARG;
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) {
        cudaGetLastError();
        return FID_ERR_NO_DEVICE;
    }
    CK(cudaSetDevice(device));
    fid_map* m = new fid_map();
    m->device = device;
    m->p = *p;
    const size_t cap = p->max_fiducials, ni = p->n_instances, wpr = (cap + 31) / 32;
    m->hash_size = 16;
    while ((size_t)m->hash_size < 2 * cap) m->hash_size *= 2;
    if (cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking) != cudaSuccess || cudaMalloc((void**)&m->d_state, sizeof(MapState) * ni) != cudaSuccess ||
        cudaMalloc((void**)&m->d_entries, sizeof(MapEntry) * ni * cap) != cudaSuccess || cudaMalloc((void**)&m->d_links, sizeof(uint32_t) * ni * cap * wpr) != cudaSuccess ||
        cudaMalloc((void**)&m->d_hash, sizeof(int32_t) * ni * 2 * (size_t)m->hash_size) != cudaSuccess ||
        cudaMalloc((void**)&m->d_export, sizeof(fid_map_record) * ni * cap) != cudaSuccess || cudaMalloc((void**)&m->d_merged, sizeof(MapEntry) * cap) != cudaSuccess ||
        cudaMalloc((void**)&m->d_merged_hdr, sizeof(MergedHeader)) != cudaSuccess || cudaMalloc((void**)&m->d_tf, sizeof(Twv) * 2) != cudaSuccess) {
        cudaGetLastError();
        fid_map_destroy(m);
        return FID_ERR_NO_MEMORY;
    }
    cudaMemset(m->d_merged_hdr, 0, sizeof(MergedHeader));
    const int rc = reset_state(m, 0, p->n_instances);
    if (rc != FID_OK) {
        fid_map_destroy(m);
        return rc;
    }
    *out = m;
    return FID_OK;
}

extern "C" int fid_map_destroy(fid_map* m) {
    if (!m) return FID_ERR_INVALID_ARG;
    cudaSetDevice(m->device);
    cudaDeviceSynchronize();
    void* ptrs[] = {m->d_var_scratch, m->d_slot_scratch, m->d_merged, m->d_merged_hdr, m->d_hash, m->d_state, m->d_entries, m->d_links, m->d_export, m->d_obs, m->d_offsets, m->d_robot, m->d_tf, m->d_merge_in, m->d_loc};
    for (void* p : ptrs)
        if (p) cudaFree(p);
    if (m->stream) cudaStreamDestroy(m->stream);
    delete m;
    return FID_OK;
}

extern "C" int fid_map_clear(fid_map* m, int instance) {
    if (!m || instance < 0 || instance >= m->p.n_instances) return FID_ERR_INVALID_ARG;
    CK(cudaSetDevice(m->device));
    CK(cudaStreamSynchronize(m->stream));
    // clearCallback (map.cpp:809-817): fiducials.clear(); initialFrameNum = frameNum; originFid = -1
    MapState st;
    CK(cudaMemcpy(&st, m->d_state + instance, sizeof(st), cudaMemcpyDeviceToHost));
    st.n = 0;
    st.initial_frame_num = st.frame_num;
    st.origin_fid = -1;
    st.initializing = 0;
    st.overflow = 0;
    st.hash_valid = 0;
    CK(cudaMemcpy(m->d_state + instance, &st, sizeof(st), cudaMemcpyHostToDevice));
    const size_t wpr = (m->p.max_fiducials + 31) / 32;
    CK(cudaMemset(m->d_links + (size_t)instance * m->p.max_fiducials * wpr, 0, sizeof(uint32_t) * (size_t)m->p.max_fiducials * wpr));
    return FID_OK;
}

extern "C" int fid_map_add_fiducial(fid_map* m, int instance, int fiducial_id, const fid_tf* T_mapBase) {
    if (!m || instance < 0 || instance >= m->p.n_instances || fiducial_id < 0) return FID_ERR_INVALID_ARG;
    CK(cudaSetDevice(m->device));
    CK(cudaStreamSynchronize(m->stream));
    MapState st;
    CK(cudaMemcpy(&st, m->d_state + instance, sizeof(st), cudaMemcpyDeviceToHost));
    st.fiducial_to_add = fiducial_id;  // addFiducialCallback (map.cpp:821-828); handled by the next update (handleAddFiducial :489-535)
    st.add_have_map_base = T_mapBase ? 1 : 0;
    if (T_mapBase) {
        for (int k = 0; k < 3; k++) st.add_map_base[k] = T_mapBase->t[k];
        for (int k = 0; k < 4; k++) st.add_map_base[3 + k] = T_mapBase->q[k];
    }
    CK(cudaMemcpy(m->d_state + instance, &st, sizeof(st), cudaMemcpyHostToDevice));
    return FID_OK;
}

static void tf_to_twv(const fid_tf& t, Twv* o) {
    q_to_m(t.q, o->R);
    o->t[0] = t.t[0];
    o->t[1] = t.t[1];
    o->t[2] = t.t[2];
    o->var = 0.0;
}

extern "C" int fid_map_load(fid_map* m, int instance, int n, const fid_map_file_entry* entries) {
    if (!m || instance < 0 || instance >= m->p.n_instances || n < 0 || (n > 0 && !entries)) return FID_ERR_INVALID_ARG;
    CK(cudaSetDevice(m->device));
    CK(cudaStreamSynchronize(m->stream));
    MapState st;
    CK(cudaMemcpy(&st, m->d_state + instance, sizeof(st), cudaMemcpyDeviceToHost));
    std::vector<MapEntry> e(st.capacity);
    if (st.n) CK(cudaMemcpy(e.data(), m->d_entries + (size_t)instance * st.capacity, sizeof(MapEntry) * st.n, cudaMemcpyDeviceToHost));
    const int lcap = m->p.max_fiducials, lwpr = (lcap + 31) / 32;
    std::vector<uint32_t> rows;
    bool rows_dirty = false;
    const double d2r = 3.14159265358979323846 / 180.0;
    for (int i = 0; i < n; i++) {
        // loadMap (map.cpp:595-606): tf2::Quaternion::setRPY(deg2rad(roll), deg2rad(pitch), deg2rad(yaw))
        const double hr = entries[i].roll_deg * d2r * 0.5, hp = entries[i].pitch_deg * d2r * 0.5, hy = entries[i].yaw_deg * d2r * 0.5;
        const double cy = cos(hy), sy = sin(hy), cp = cos(hp), sp = sin(hp), cr = cos(hr), sr = sin(hr);
        const double q[4] = {sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy};
        int slot = -1;
        for (int j = 0; j < st.n; j++)
            if (e[j].id == entries[i].fiducial_id) slot = j;
        if (slot < 0) {
            if (st.n >= st.capacity) return FID_ERR_CAPACITY;
            slot = st.n++;
        } else {
            if (rows.empty()) {
                rows.resize((size_t)lcap * lwpr);
                CK(cudaMemcpy(rows.data(), m->d_links + (size_t)instance * lcap * lwpr, sizeof(uint32_t) * rows.size(), cudaMemcpyDeviceToHost));
            }
            for (int w = 0; w < lwpr; w++) rows[(size_t)slot * lwpr + w] = 0;                                     // its own links
            for (int j = 0; j < lcap; j++) rows[(size_t)j * lwpr + (slot >> 5)] &= ~(1u << (slot & 31));          // links to it
            rows_dirty = true;
        }
        e[slot].id = entries[i].fiducial_id;
        e[slot].num_obs = entries[i].num_obs;
        q_to_m(q, e[slot].pose.R);
        e[slot].pose.t[0] = entries[i].x;
        e[slot].pose.t[1] = entries[i].y;
        e[slot].pose.t[2] = entries[i].z;
        e[slot].pose.var = entries[i].variance;
    }
    st.hash_valid = 0;
    if (st.n) CK(cudaMemcpy(m->d_entries + (size_t)instance * st.capacity, e.data(), sizeof(MapEntry) * st.n, cudaMemcpyHostToDevice));
    if (rows_dirty) CK(cudaMemcpy(m->d_links + (size_t)instance * lcap * lwpr, rows.data(), sizeof(uint32_t) * rows.size(), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(m->d_state + instance, &st, sizeof(st), cudaMemcpyHostToDevice));
    return FID_OK;
}

template <class T>
static int ensure(T** p, size_t* cap, size_t need) {
    if (need <= *cap) return FID_OK;
    if (*p) cudaFree(*p);
    *p = nullptr;
    *cap = 0;
    const size_t n = std::max<size_t>(need, 1024);
    if (cudaMalloc((void**)p, sizeof(T) * n) != cudaSuccess) {
        cudaGetLastError();
        return FID_ERR_NO_MEMORY;
    }
    *cap = n;
    return FID_OK;
}

static int run_sequence(fid_map* m, int inst_lo, int n_inst, int n_msgs, const int32_t* offsets, const fid_transform* obs, const fid_tf* T_baseCam,
                        const fid_tf* T_camBase, fid_robot_pose* robot, bool async = false) {
    CK(cudaSetDevice(m->device));
    CK(cudaStreamSynchronize(m->stream));  // a pending asynchronous update still owns the staging buffers
    const size_t n_off = (size_t)n_inst * (n_msgs + 1);
    size_t total_obs = 0;
    for (size_t i = 0; i < n_off; i++) total_obs = std::max<size_t>(total_obs, (size_t)offsets[i]);
    int rc;
    if ((rc = ensure(&m->d_obs, &m->obs_cap, total_obs + 1)) != FID_OK || (rc = ensure(&m->d_var_scratch, &m->var_cap, total_obs + 1)) != FID_OK ||
        (rc = ensure(&m->d_slot_scratch, &m->slot_cap, total_obs + 1)) != FID_OK || (rc = ensure(&m->d_offsets, &m->off_cap, n_off)) != FID_OK ||
        (rc = ensure(&m->d_robot, &m->robot_cap, (size_t)n_inst * n_msgs + 1)) != FID_OK)
        return rc;
    std::vector<Obs> ho(total_obs);
    for (size_t i = 0; i < total_obs; i++) {
        ho[i].id = obs[i].fiducial_id;
        ho[i].pad = 0;
        for (int k = 0; k < 3; k++) ho[i].t[k] = obs[i].translation[k];
        for (int k = 0; k < 4; k++) ho[i].q[k] = obs[i].rotation[k];
        ho[i].object_error = obs[i].object_error;
        ho[i].area = obs[i].fiducial_area;
    }
    // (pageable sources: the runtime stages these copies before returning, so the host vectors may die)
    if (total_obs) CK(cudaMemcpyAsync(m->d_obs, ho.data(), sizeof(Obs) * total_obs, cudaMemcpyHostToDevice, m->stream));
    CK(cudaMemcpyAsync(m->d_offsets, offsets, sizeof(int32_t) * n_off, cudaMemcpyHostToDevice, m->stream));
    Twv tf[2];
    memset(tf, 0, sizeof(tf));
    if (T_baseCam) tf_to_twv(*T_baseCam, &tf[0]);
    if (T_camBase) tf_to_twv(*T_camBase, &tf[1]);
    CK(cudaMemcpyAsync(m->d_tf, tf, sizeof(tf), cudaMemcpyHostToDevice, m->stream));
    SeqArgs a{};
    const int cap = m->p.max_fiducials;
    a.state = m->d_state + inst_lo;
    a.entries = m->d_entries + (size_t)inst_lo * cap;
    a.links_wpr = (cap + 31) / 32;
    a.links = m->d_links + (size_t)inst_lo * cap * a.links_wpr;
    a.cap = cap;
    a.hash = m->d_hash + (size_t)inst_lo * 2 * m->hash_size;
    a.hash_size = m->hash_size;
    a.n_instances = n_inst;
    a.n_msgs = n_msgs;
    a.offsets = m->d_offsets;
    a.obs = m->d_obs;
    a.var_scratch = m->d_var_scratch;
    a.slot_scratch = m->d_slot_scratch;
    a.tf = m->d_tf;
    a.have_base_cam = T_baseCam ? 1 : 0;
    a.have_cam_base = T_camBase ? 1 : 0;
    a.weighting_scale = m->p.weighting_scale;
    a.systematic_error = m->p.systematic_error;
    a.use_area = m->p.use_fiducial_area_as_weight;
    a.robot = m->d_robot;
    k_map_sequence<<<(n_inst + 31) / 32, 32, 0, m->stream>>>(a);
    CK(cudaGetLastError());
    if (async) return FID_OK;
    std::vector<RobotPose> hr((size_t)n_inst * n_msgs);
    CK(cudaMemcpyAsync(hr.data(), m->d_robot, sizeof(RobotPose) * hr.size(), cudaMemcpyDeviceToHost, m->stream));
    CK(cudaStreamSynchronize(m->stream));
    if (robot)
        for (size_t i = 0; i < hr.size(); i++) {
            robot[i].valid = hr[i].valid;
            robot[i].n_estimates = hr[i].n_estimates;
            for (int k = 0; k < 3; k++) robot[i].t[k] = hr[i].t[k];
            for (int k = 0; k < 4; k++) robot[i].q[k] = hr[i].q[k];
            robot[i].variance = hr[i].var;
        }
    return FID_OK;
}

extern "C" int fid_map_update(fid_map* m, int instance, int n_obs, const fid_transform* obs, const fid_tf* T_baseCam, const fid_tf* T_camBase, fid_robot_pose* robot) {
    if (!m || instance < 0 || instance >= m->p.n_instances || n_obs < 0 || (n_obs > 0 && !obs)) return FID_ERR_INVALID_ARG;
    const int32_t off[2] = {0, n_obs};
    return run_sequence(m, instance, 1, 1, off, obs, T_baseCam, T_camBase, robot);
}

extern "C" int fid_map_update_sequence(fid_map* m, int n_msgs, const int32_t* offsets, const fid_transform* obs, const fid_tf* T_baseCam, const fid_tf* T_camBase,
                                       fid_robot_pose* robot) {
    if (!m || n_msgs < 1 || !offsets) return FID_ERR_INVALID_ARG;
    const size_t n_off = (size_t)m->p.n_instances * (n_msgs + 1);
    for (size_t i = 0; i + 1 < n_off; i++) {
        if ((i + 1) % (n_msgs + 1) == 0) continue;
        const int d = offsets[i + 1] - offsets[i];
        if (d < 0) return FID_ERR_INVALID_ARG;
    }
    return run_sequence(m, 0, m->p.n_instances, n_msgs, offsets, obs, T_baseCam, T_camBase, robot);
}

static int update_frames_impl(fid_map* m, int instance, int n_frames, const int32_t* counts, const fid_transform* transforms, int max_markers, const fid_tf* T_baseCam,
                              const fid_tf* T_camBase, fid_robot_pose* last_robot, bool async) {
    if (!m || instance < 0 || instance >= m->p.n_instances || n_frames < 1 || !counts || !transforms || max_markers < 1) return FID_ERR_INVALID_ARG;
    std::vector<int32_t> off((size_t)n_frames + 1, 0);
    std::vector<fid_transform> flat;
    for (int f = 0; f < n_frames; f++) {
        const int c = std::min(std::max(counts[f], 0), max_markers);  // every observation of the frame (a message has no size limit, map.cpp:152)
        off[f] = (int32_t)flat.size();
        flat.insert(flat.end(), transforms + (size_t)f * max_markers, transforms + (size_t)f * max_markers + c);
    }
    off[n_frames] = (int32_t)flat.size();
    std::vector<fid_robot_pose> robots((size_t)n_frames);
    fid_transform dummy{};
    const int rc = run_sequence(m, instance, 1, n_frames, off.data(), flat.empty() ? &dummy : flat.data(), T_baseCam, T_camBase, async ? nullptr : robots.data(), async);
    if (rc == FID_OK && last_robot && !async) *last_robot = robots[(size_t)n_frames - 1];
    return rc;
}

extern "C" int fid_map_update_frames(fid_map* m, int instance, int n_frames, const int32_t* counts, const fid_transform* transforms, int max_markers, const fid_tf* T_baseCam,
                                     const fid_tf* T_camBase, fid_robot_pose* last_robot) {
    return update_frames_impl(m, instance, n_frames, counts, transforms, max_markers, T_baseCam, T_camBase, last_robot, false);
}
extern "C" int fid_map_update_frames_async(fid_map* m, int instance, int n_frames, const int32_t* counts, const fid_transform* transforms, int max_markers,
                                           const fid_tf* T_baseCam, const fid_tf* T_camBase) {
    return update_frames_impl(m, instance, n_frames, counts, transforms, max_markers, T_baseCam, T_camBase, nullptr, true);
}
extern "C" int fid_map_sync(fid_map* m) {
    if (!m) return FID_ERR_INVALID_ARG;
    CK(cudaSetDevice(m->device));
    CK(cudaStreamSynchronize(m->stream));
    return FID_OK;
}

extern "C" int fid_map_entries(fid_map* m, int instance, int max_entries, int* n, fid_map_entry* entries) {
    if (!m || instance < 0 || instance >= m->p.n_instances || !n) return FID_ERR_INVALID_ARG;
    CK(cudaSetDevice(m->device));
    CK(cudaStreamSynchronize(m->stream));
    MapState st;
    CK(cudaMemcpy(&st, m->d_state + instance, sizeof(st), cudaMemcpyDeviceToHost));
    std::vector<MapEntry> e(st.n);
    if (st.n) CK(cudaMemcpy(e.data(), m->d_entries + (size_t)instance * st.capacity, sizeof(MapEntry) * st.n, cudaMemcpyDeviceToHost));
    std::sort(e.begin(), e.end(), [](const MapEntry& a, const MapEntry& b) { return a.id < b.id; });
    *n = st.n;
    if (st.n > max_entries) return FID_ERR_CAPACITY;
    for (int i = 0; i < st.n && entries; i++) {
        // publishMap (map.cpp:629-654): origin + getRPY
        entries[i].fiducial_id = e[i].id;
        entries[i].num_obs = e[i].num_obs;
        entries[i].x = e[i].pose.t[0];
        entries[i].y = e[i].pose.t[1];
        entries[i].z = e[i].pose.t[2];
        get_rpy(e[i].pose.R, &entries[i].rx, &entries[i].ry, &entries[i].rz);
        entries[i].variance = e[i].pose.var;
    }
    return st.overflow ? FID_ERR_CAPACITY : FID_OK;
}

// links (map.cpp:217-222, saved by saveMap :557-559): the device keeps them as a slot x slot bit matrix.
extern "C" int fid_map_links(fid_map* m, int instance, int max_pairs, int* n_pairs, int32_t* pairs) {
    if (!m || instance < 0 || instance >= m->p.n_instances || !n_pairs || max_pairs < 0) return FID_ERR_INVALID_ARG;
    CK(cudaSetDevice(m->device));
    CK(cudaStreamSynchronize(m->stream));
    MapState st;
    CK(cudaMemcpy(&st, m->d_state + instance, sizeof(st), cudaMemcpyDeviceToHost));
    const int cap = m->p.max_fiducials, wpr = (cap + 31) / 32;
    std::vector<MapEntry> e(st.n);
    std::vector<uint32_t> rows((size_t)st.n * wpr);
    if (st.n) {
        CK(cudaMemcpy(e.data(), m->d_entries + (size_t)instance * st.capacity, sizeof(MapEntry) * st.n, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(rows.data(), m->d_links + (size_t)instance * cap * wpr, sizeof(uint32_t) * rows.size(), cudaMemcpyDeviceToHost));
    }
    std::vector<std::pair<int32_t, int32_t>> out;
    for (int i = 0; i < st.n; i++)
        for (int j = 0; j < st.n; j++)
            if ((rows[(size_t)i * wpr + (j >> 5)] >> (j & 31)) & 1u) out.emplace_back(e[i].id, e[j].id);
    std::sort(out.begin(), out.end());  // std::map<int, Fiducial> / std::set<int> links iterate ascending
    *n_pairs = (int)out.size();
    if ((int)out.size() > max_pairs) return FID_ERR_CAPACITY;
    for (size_t k = 0; k < out.size() && pairs; k++) {
        pairs[2 * k] = out[k].first;
        pairs[2 * k + 1] = out[k].second;
    }
    return FID_OK;
}

extern "C" int fid_map_add_links(fid_map* m, int instance, int n_pairs, const int32_t* pairs) {
    if (!m || instance < 0 || instance >= m->p.n_instances || n_pairs < 0 || (n_pairs > 0 && !pairs)) return FID_ERR_INVALID_ARG;
    if (n_pairs == 0) return FID_OK;
    CK(cudaSetDevice(m->device));
    CK(cudaStreamSynchronize(m->stream));
    MapState st;
    CK(cudaMemcpy(&st, m->d_state + instance, sizeof(st), cudaMemcpyDeviceToHost));
    const int cap = m->p.max_fiducials, wpr = (cap + 31) / 32;
    std::vector<MapEntry> e(st.n);
    std::vector<uint32_t> rows((size_t)st.n * wpr);
    if (!st.n) return FID_OK;
    CK(cudaMemcpy(e.data(), m->d_entries + (size_t)instance * st.capacity, sizeof(MapEntry) * st.n, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(rows.data(), m->d_links + (size_t)instance * cap * wpr, sizeof(uint32_t) * rows.size(), cudaMemcpyDeviceToHost));
    auto slot_of = [&](int32_t id) {
        for (int i = 0; i < st.n; i++)
            if (e[i].id == id) return i;
        return -1;
    };
    for (int k = 0; k < n_pairs; k++) {
        const int i = slot_of(pairs[2 * k]), j = slot_of(pairs[2 * k + 1]);
        if (i >= 0 && j >= 0) rows[(size_t)i * wpr + (j >> 5)] |= 1u << (j & 31);  // a link to a fiducial that is not in the map cannot be kept
    }
    CK(cudaMemcpy(m->d_links + (size_t)instance * cap * wpr, rows.data(), sizeof(uint32_t) * rows.size(), cudaMemcpyHostToDevice));
    return FID_OK;
}

static int launch_export(fid_map* m, int instance, fid_map_record* dst) {
    k_map_export<<<1, 256, 0, m->stream>>>(m->d_state, m->d_entries, m->p.max_fiducials, instance, dst);
    CK(cudaGetLastError());
    return FID_OK;
}

extern "C" int fid_map_export_device(fid_map* m, int instance, void** device_table, size_t* bytes) {
    if (!m || instance < 0 || instance >= m->p.n_instances || !device_table || !bytes) return FID_ERR_INVALID_ARG;
    CK(cudaSetDevice(m->device));
    fid_map_record* tab = m->d_export + (size_t)instance * m->p.max_fiducials;
    const int rc = launch_export(m, instance, tab);
    if (rc != FID_OK) return rc;
    CK(cudaStreamSynchronize(m->stream));
    *device_table = tab;
    *bytes = sizeof(fid_map_record) * (size_t)m->p.max_fiducials;
    return FID_OK;
}

extern "C" int fid_map_export_async(fid_map* m, int instance, void* device_dst) {
    if (!m || instance < 0 || instance >= m->p.n_instances || !device_dst) return FID_ERR_INVALID_ARG;
    CK(cudaSetDevice(m->device));
    return launch_export(m, instance, (fid_map_record*)device_dst);  // ordered after pending updates on the map's stream
}

extern "C" int fid_map_export(fid_map* m, int instance, fid_map_record* table) {
    if (!table) return FID_ERR_INVALID_ARG;
    void* d = nullptr;
    size_t bytes = 0;
    const int rc = fid_map_export_device(m, instance, &d, &bytes);
    if (rc != FID_OK) return rc;
    CK(cudaMemcpy(table, d, bytes, cudaMemcpyDeviceToHost));
    return FID_OK;
}

extern "C" int fid_map_stream(fid_map* m, void** cuda_stream) {
    if (!m || !cuda_stream) return FID_ERR_INVALID_ARG;
    *cuda_stream = (void*)m->stream;
    return FID_OK;
}

extern "C" int fid_map_merge_device_async(fid_map* m, int n_tables, const void* device_tables) {
    if (!m || n_tables < 1 || !device_tables) return FID_ERR_INVALID_ARG;
    CK(cudaSetDevice(m->device));
    const int cap = m->p.max_fiducials;
    if ((long long)n_tables * cap <= MERGE_MAX_KEYS)
        k_map_merge_view<<<1, 1024, 0, m->stream>>>(cap, n_tables, (const fid_map_record*)device_tables, m->d_merged, m->d_merged_hdr);
    else
        k_map_merge_view_serial<<<1, 32, 0, m->stream>>>(cap, n_tables, (const fid_map_record*)device_tables, m->d_merged, m->d_merged_hdr);
    CK(cudaGetLastError());
    return FID_OK;
}

extern "C" int fid_map_merge_device(fid_map* m, int n_tables, const void* device_tables) {
    const int rc = fid_map_merge_device_async(m, n_tables, device_tables);
    if (rc != FID_OK) return rc;
    CK(cudaStreamSynchronize(m->stream));
    return FID_OK;
}

extern "C" int fid_map_merge(fid_map* m, int n_tables, const fid_map_record* tables) {
    if (!m || n_tables < 1 || !tables) return FID_ERR_INVALID_ARG;
    CK(cudaSetDevice(m->device));
    CK(cudaStreamSynchronize(m->stream));  // an earlier asynchronous merge may still read the staging buffer
    const size_t need = (size_t)n_tables * m->p.max_fiducials;
    const int rc = ensure(&m->d_merge_in, &m->merge_cap, need);
    if (rc != FID_OK) return rc;
    CK(cudaMemcpyAsync(m->d_merge_in, tables, sizeof(fid_map_record) * need, cudaMemcpyHostToDevice, m->stream));
    return fid_map_merge_device(m, n_tables, m->d_merge_in);
}

extern "C" int fid_map_merged_entries(fid_map* m, int max_entries, int* n, fid_map_entry* entries) {
    if (!m || !n || max_entries < 0) return FID_ERR_INVALID_ARG;
    CK(cudaSetDevice(m->device));
    CK(cudaStreamSynchronize(m->stream));
    MergedHeader hdr;
    CK(cudaMemcpy(&hdr, m->d_merged_hdr, sizeof(hdr), cudaMemcpyDeviceToHost));
    *n = hdr.n;
    if (hdr.n > max_entries) return FID_ERR_CAPACITY;
    std::vector<MapEntry> e(hdr.n);
    if (hdr.n) CK(cudaMemcpy(e.data(), m->d_merged, sizeof(MapEntry) * hdr.n, cudaMemcpyDeviceToHost));
    for (int i = 0; i < hdr.n && entries; i++) {
        entries[i].fiducial_id = e[i].id;
        entries[i].num_obs = e[i].num_obs;
        entries[i].x = e[i].pose.t[0];
        entries[i].y = e[i].pose.t[1];
        entries[i].z = e[i].pose.t[2];
        get_rpy(e[i].pose.R, &entries[i].rx, &entries[i].ry, &entries[i].rz);
        entries[i].variance = e[i].pose.var;
    }
    return hdr.overflow ? FID_ERR_CAPACITY : FID_OK;
}

extern "C" int fid_map_adopt_merged(fid_map* m, int instance) {
    if (!m || instance < 0 || instance >= m->p.n_instances) return FID_ERR_INVALID_ARG;
    CK(cudaSetDevice(m->device));
    const int cap = m->p.max_fiducials;
    k_map_adopt<<<1, 256, 0, m->stream>>>(m->d_state, m->d_entries, m->d_links, cap, (cap + 31) / 32, instance, m->d_merged, m->d_merged_hdr);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(m->stream));
    return FID_OK;
}
