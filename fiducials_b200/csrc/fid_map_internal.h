// Internal state of a map handle, shared by fid_map.cu (sequential fold, merged view) and fid_map_refine.cu (batch refinement).
#pragma once
#include <cuda_runtime.h>
#include <stdio.h>

#include "../../include/fiducials_b200.h"
#include "slam.cuh"

#ifndef CK
#define CK(call)                                                                                       \
    do {                                                                                               \
        cudaError_t e_ = (call);                                                                       \
        if (e_ != cudaSuccess) {                                                                       \
            fprintf(stderr, "[fiducials_b200] CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); \
            return FID_ERR_CUDA;                                                                       \
        }                                                                                              \
    } while (0)
#endif

struct fid_map {
    int device = 0;
    fid_map_params p{};
    cudaStream_t stream = nullptr;
    fid::MapState* d_state = nullptr;      // [n_instances]
    fid::MapEntry* d_entries = nullptr;    // [n_instances][cap]
    uint32_t* d_links = nullptr;      // [n_instances][cap][ceil(cap/32)]
    int32_t* d_hash = nullptr;        // [n_instances][2][hash_size]  id -> slot
    int hash_size = 0;
    fid_map_record* d_export = nullptr;  // [n_instances][cap]
    fid::Obs* d_obs = nullptr;
    size_t obs_cap = 0;
    double* d_var_scratch = nullptr;  // per observation: updatePose's variance write-back (map.cpp:298)
    size_t var_cap = 0;
    int* d_slot_scratch = nullptr;    // per observation: map slot (link pass)
    size_t slot_cap = 0;
    int32_t* d_offsets = nullptr;
    size_t off_cap = 0;
    fid::RobotPose* d_robot = nullptr;
    size_t robot_cap = 0;
    fid::Twv* d_tf = nullptr;  // [2]: baseCam, camBase
    fid_map_record* d_merge_in = nullptr;
    size_t merge_cap = 0;
    fid::MapEntry* d_merged = nullptr;     // [cap] merged view (ids ascending)
    struct MergedHeader* d_merged_hdr = nullptr;
    char* d_loc = nullptr;                 // fid_map_localize: inputs, per-frame scratch and results (grown by the call)
    size_t loc_cap = 0;
};

