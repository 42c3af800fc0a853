/* fiducials_b200 -- C ABI of libfiducials_b200.so
 *
 * H100-native (sm_90a) replacement for the per-frame hot path of UbiquityRobotics/fiducials:
 *   aruco_detect  : cv::aruco::detectMarkers + per-marker cv::solvePnP + message arithmetic
 *   fiducial_slam : Map::update (pose fold + map fusion)
 *
 * The reference has no plugin/FFI interface; the seam is three OpenCV call sites and Map::update
 * (SURVEY.md 8b).  Each entry point below cites the reference code it replaces (paths relative to the
 * reference repository).  Conventions: plain C, caller owns every host array, every function returns
 * an int status (FID_OK == 0, negative = error, see fid_strerror), nothing throws across the boundary,
 * n == 0 markers is a valid result.  A handle is single-caller (the reference processes one callback
 * at a time, aruco_detect.cpp:737); concurrency = several handles or the batch calls.
 * There is NO CPU fallback: fid_create fails with FID_ERR_NO_DEVICE when no CUDA device is usable.
 */
#ifndef FIDUCIALS_B200_H
#define FIDUCIALS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FID_OK 0
#define FID_ERR_INVALID_ARG (-1)
#define FID_ERR_NO_DEVICE (-2)
#define FID_ERR_CUDA (-3)
#define FID_ERR_UNSUPPORTED (-4) /* dictionary / parameter outside the implemented range */
#define FID_ERR_CAPACITY (-5)    /* an internal or caller-provided buffer was too small */
#define FID_ERR_NO_MEMORY (-6)

const char* fid_strerror(int status);
/* Library version "major.minor.patch". */
const char* fid_version(void);

/* ------------------------------------------------------------------------------------------------
 * Detector parameters.  Field-for-field the values FiducialsNode sets on
 * cv::aruco::DetectorParameters (aruco_detect/src/aruco_detect.cpp:690-727, same list as
 * aruco_detect/cfg/DetectorParams.cfg), the dictionary enum (aruco_detect.cpp:611,671) and the two
 * OpenCV >= 4.7 fields that exist only in the oracle's OpenCV (SURVEY.md A.0).
 * ---------------------------------------------------------------------------------------------- */
typedef struct fid_params {
    int32_t dictionary;                        /* OpenCV enum: 4..7 = DICT_5X5_{50,100,250,1000}, 8..11 = DICT_6X6_* ; default 7 (:611) */
    double adaptiveThreshConstant;             /* 7      (:690) */
    int32_t adaptiveThreshWinSizeMax;          /* 53     (:691) */
    int32_t adaptiveThreshWinSizeMin;          /* 3      (:692) */
    int32_t adaptiveThreshWinSizeStep;         /* 4      (:693) */
    int32_t cornerRefinementMaxIterations;     /* 30     (:694) */
    double cornerRefinementMinAccuracy;        /* 0.01   (:695) */
    int32_t cornerRefinementWinSize;           /* 5      (:696) */
    int32_t cornerRefinementMethod;            /* 0 NONE, 1 SUBPIX (default), 2 CONTOUR (doCornerRefinement / cornerRefinementSubPix, :700-711) */
    double errorCorrectionRate;                /* 0.6    (:716) */
    double minCornerDistanceRate;              /* 0.05   (:717) */
    int32_t markerBorderBits;                  /* 1      (:718) */
    double maxErroneousBitsInBorderRate;       /* 0.04   (:719) */
    int32_t minDistanceToBorder;               /* 3      (:720) */
    double minMarkerDistanceRate;              /* 0.05   (:721) */
    double minMarkerPerimeterRate;             /* 0.1    (:722) */
    double maxMarkerPerimeterRate;             /* 4.0    (:723) */
    double minOtsuStdDev;                      /* 5.0    (:724) */
    double perspectiveRemoveIgnoredMarginPerCell; /* 0.13 (:725) */
    int32_t perspectiveRemovePixelPerCell;     /* 8      (:726) */
    double polygonalApproxAccuracyRate;        /* 0.01   (:727) */
    double relativeCornerRefinmentWinSize;     /* OpenCV>=4.7 only; 100 reproduces the reference's OpenCV (SURVEY P4) */
    double minGroupDistance;                   /* OpenCV>=4.7 only; 0.21 */
} fid_params;

/* Fill *p with the reference's rosparam defaults (aruco_detect.cpp:609-727). */
int fid_default_params(fid_params* p);

/* ------------------------------------------------------------------------------------------------
 * Detector handle.  Replaces `new aruco::DetectorParameters` (aruco_detect.cpp:607) +
 * aruco::getPredefinedDictionary(dicno) (:671).  Owns device buffers for `max_batch` frames of up
 * to max_width x max_height BGR8 pixels, the CUDA streams and the dictionary tables.
 * ---------------------------------------------------------------------------------------------- */
typedef struct fid_detector fid_detector;

int fid_create(const fid_params* params, int device, int max_width, int max_height, int max_batch, fid_detector** out);
int fid_destroy(fid_detector* h);
/* configCallback (aruco_detect.cpp:257-298): change parameters between frames. */
int fid_set_params(fid_detector* h, const fid_params* params);

#define FID_MAX_MARKERS 256 /* per frame */

/* One frame, detect only.  Replaces cv::aruco::detectMarkers(image, dictionary, corners, ids,
 * detectorParams) at aruco_detect.cpp:350.  bgr = H x W x 3 uint8 host pixels (what
 * cv_bridge::toCvCopy(msg, BGR8) yields, :348), `stride` bytes per row.  Outputs (host arrays of
 * capacity max_markers): ids[n], corners[n*8] = x0,y0..x3,y3 in OpenCV's corner order and OpenCV's
 * marker order -- exactly what imageCallback copies into fiducial_msgs/Fiducial (:358-377). */
int fid_detect(fid_detector* h, const uint8_t* bgr, int width, int height, size_t stride, int max_markers, int* n, int32_t* ids, float* corners);

/* Camera intrinsics as latched by camInfoCallback (aruco_detect.cpp:307-330): K row-major 3x3,
 * D = first five plumb_bob coefficients k1 k2 p1 p2 k3. */
typedef struct fid_camera {
    double K[9];
    double D[5];
} fid_camera;

/* Per-marker pose record = the fields of fiducial_msgs/FiducialTransform
 * (fiducial_msgs/msg/FiducialTransform.msg:2-6) plus the raw rvec (needed for parity checks). */
typedef struct fid_transform {
    int32_t fiducial_id;
    int32_t reserved;
    double translation[3];  /* tvec                                   (aruco_detect.cpp:481-483) */
    double rotation[4];     /* quaternion x,y,z,w from axis/angle      (:447-448, :485-489) */
    double image_error;     /* mean squared reprojection error, px^2   (:203-221, :491) */
    double object_error;    /* (:493-495) */
    double fiducial_area;   /* Heron area of the quad, px^2            (:179-200, :490) */
    double rvec[3];         /* raw SOLVEPNP_ITERATIVE output, not wrapped */
} fid_transform;

/* Pose for markers already detected.  Replaces estimatePoseSingleMarkers (aruco_detect.cpp:223-255:
 * getSingleMarkerObjectPoints :151-161 + cv::solvePnP :247 + getReprojectionError :203-221) and the
 * per-marker arithmetic of poseEstimateCallback (:447-495).  fiducial_len is the node's
 * `fiducial_len` (:615); (override_ids, override_lens, n_override) mirror `fiducial_len_override`
 * (:627-660).  Like the reference, object_error always uses fiducial_len, not the override. */
int fid_pose(fid_detector* h, int n, const int32_t* ids, const float* corners, const fid_camera* cam, double fiducial_len, int n_override,
             const int32_t* override_ids, const double* override_lens, fid_transform* out);

/* Batched detect + pose: n_frames frames of identical size.  Frame f occupies
 * bgr + f*frame_stride bytes.  Outputs: counts[f] markers; ids/corners/transforms are dense
 * [n_frames][max_markers] arrays.  `bgr_on_device` != 0 means `bgr` is a device pointer already in
 * HBM (used by bench.py's device-resident figure); otherwise it is (ideally pinned) host memory
 * and the copy is part of the call.  Results always land in host arrays. */
int fid_detect_pose_batch(fid_detector* h, int n_frames, const uint8_t* bgr, int bgr_on_device, int width, int height, size_t row_stride, size_t frame_stride,
                          const fid_camera* cam, double fiducial_len, int n_override, const int32_t* override_ids, const double* override_lens,
                          int max_markers, int32_t* counts, int32_t* ids, float* corners, fid_transform* transforms);

/* The same call split in two, for a camera stream: fid_submit_batch queues the uploads and kernels of a
 * batch and returns at once; fid_collect_batch waits for the OLDEST submitted batch and writes its results
 * (same layout as fid_detect_pose_batch).  While batch k finishes its latency-bound tail (grouping,
 * identification, pose) batch k+1 already runs its threshold and border-walk stages -- the reference
 * node has the same structure between its image callback and its publishers, one frame at a time.
 * A batch needs ceil(n_frames / max_batch) free chunk slots; the handle has 4 of them (environment
 * FID_SLOTS, 2..8).  FID_ERR_CAPACITY = not enough free slots, collect first.  The frames of
 * a host `bgr` must stay valid and unchanged until the batch has been collected.
 * fid_detect_pose_batch may only be called while nothing is in flight. */
int fid_submit_batch(fid_detector* h, int n_frames, const uint8_t* bgr, int bgr_on_device, int width, int height, size_t row_stride, size_t frame_stride,
                     const fid_camera* cam, double fiducial_len, int n_override, const int32_t* override_ids, const double* override_lens);
int fid_collect_batch(fid_detector* h, int max_markers, int32_t* counts, int32_t* ids, float* corners, fid_transform* transforms);

/* Pixel format of the frames handed to every entry point that takes `bgr` (default FID_ENC_BGR8).  The
 * reference converts whatever the camera publishes with cv_bridge::toCvCopy(msg, BGR8)
 * (aruco_detect.cpp:348) before detectMarkers turns it into gray again; the library takes the camera's own
 * encoding and produces the identical gray plane: RGB8 = channels swapped, MONO8 = the plane itself (one
 * byte per pixel: a third of the upload).  Strides are in bytes of that encoding.  Not while batches are
 * in flight. */
enum { FID_ENC_BGR8 = 0, FID_ENC_RGB8 = 1, FID_ENC_MONO8 = 2 };
int fid_set_input_encoding(fid_detector* h, int encoding);

/* Streaming hint: `next_bgr` (pinned host memory, same frame count and geometry as the call that
 * follows this hint) will be the `bgr` argument of the call after that one.  The library then
 * uploads its first chunk in the background once the uploads of the call in progress are queued, so
 * the next call does not start with an exposed H2D copy.  The frames must not change between the
 * hinted call and their own call.  Passing NULL clears the hint. */
int fid_hint_next(fid_detector* h, const uint8_t* next_bgr);

/* Device-side stopwatch for benchmarks: start records a CUDA event on the handle's compute stream,
 * stop records a second one, waits for it and returns the elapsed milliseconds between the two. */
int fid_timer_start(fid_detector* h);
int fid_timer_stop(fid_detector* h, float* elapsed_ms);

/* Pinned host memory helpers for callers that want the async copy path. */
int fid_host_alloc(size_t bytes, void** out);
int fid_host_free(void* p);
int fid_device_alloc(fid_detector* h, size_t bytes, void** out);
int fid_device_free(fid_detector* h, void* p);
int fid_memcpy_h2d(fid_detector* h, void* dst_device, const void* src_host, size_t bytes);

/* Stage access for parity tests and profiling (device results copied to host).
 *   gray:   H x W uint8 (cvtColor BGR2GRAY)
 *   planes: n_scales x H x W uint8 {0,1} (adaptiveThreshold per window size)
 * Runs only the threshold stage on one frame. */
int fid_debug_threshold(fid_detector* h, const uint8_t* bgr, int width, int height, size_t stride, uint8_t* gray, uint8_t* planes, int* n_scales);
/* Profiling aid: runs ONLY the threshold stage (k_gray + k_threshold) `reps` times on n_frames
 * device-resident frames (n_frames <= max_batch), nothing else on the GPU, and returns the average device
 * time of one pass in milliseconds (CUDA events on the launching stream).  bench.py reports the stage's
 * roofline fraction from this figure next to the one measured inside the pipelined step. */
int fid_debug_time_threshold(fid_detector* h, int n_frames, const uint8_t* bgr_device, int width, int height, size_t row_stride, size_t frame_stride, int reps,
                             float* ms_per_pass);
/* Quad candidates of the last fid_detect call on slot 0, in OpenCV's concatenation order
 * (scale-major, contour-list order): quads[n*8] int32 vertices (approxPolyDP order), scale[n],
 * contour_len[n]. */
int fid_debug_candidates(fid_detector* h, int max_candidates, int* n, int32_t* quads, int32_t* scale, int32_t* contour_len);

/* Per-stage device times (milliseconds, CUDA events) of the last batch call:
 * [0] h2d copy, [1] threshold (+ start cracks), [2] unused (reads 0), [3] border walk, [4] chain emit, [5] polygon+filters,
 * [6] group, [7] identify, [8] subpix+pose, [9] unused, [10] d2h, [11..18] the border-walk rounds
 * (unused rounds read 0); n_stages returns 19. */
int fid_last_stage_ms(fid_detector* h, float* ms, int max_stages, int* n_stages);
/* Work counters of the last batch call: [0] start cracks, [1] walk survivors (contours in range),
 * [2] contour points emitted, [3] quad candidates, [4] candidates selected, [5] markers,
 * [6] kernel launches issued. */
int fid_last_counters(fid_detector* h, int64_t* counters, int max_counters, int* n_counters);

/* ------------------------------------------------------------------------------------------------
 * Map / fiducial_slam.  State mirrors Map (fiducial_slam/include/fiducial_slam/map.h:118-134):
 * fiducials, frameNum, initialFrameNum, originFid, isInitializingMap, readOnly.
 * ---------------------------------------------------------------------------------------------- */
typedef struct fid_map fid_map;

typedef struct fid_map_params {
    double weighting_scale;           /* 1e9   (fiducial_slam.cpp:115) */
    int32_t use_fiducial_area_as_weight; /* 0  (fiducial_slam.cpp:113) */
    int32_t read_only_map;            /* 0     (map.cpp:129) */
    double systematic_error;          /* 0.01  (map.cpp:50) */
    int32_t max_fiducials;            /* table capacity per map instance */
    int32_t n_instances;              /* independent map instances held by this handle (one per camera stream) */
} fid_map_params;

int fid_map_default_params(fid_map_params* p);
int fid_map_create(const fid_map_params* p, int device, fid_map** out);
int fid_map_destroy(fid_map* m);
/* clearCallback (map.cpp:809-817). */
int fid_map_clear(fid_map* m, int instance);

/* One line of the map file (map.cpp:556-562 / loadMap :595-606): angles in DEGREES as in the file. */
typedef struct fid_map_file_entry {
    int32_t fiducial_id;
    int32_t num_obs;
    double x, y, z, roll_deg, pitch_deg, yaw_deg, variance;
} fid_map_file_entry;
int fid_map_load(fid_map* m, int instance, int n, const fid_map_file_entry* entries);

/* The link sets of the map (Fiducial::links, map.h:87; filled by updateMap map.cpp:217-222, written after
 * numObs on every line of the map file, saveMap :557-559 / loadMap :608-615) as (fiducial_id, linked_id) pairs in
 * ascending order.  fid_map_add_links is the loadMap direction; a link to an id that is not in the map is dropped. */
int fid_map_links(fid_map* m, int instance, int max_pairs, int* n_pairs, int32_t* pairs);
int fid_map_add_links(fid_map* m, int instance, int n_pairs, const int32_t* pairs);

/* 7-vector transform: x y z qx qy qz qw (what the host obtains from tf, map.cpp:258-273). */
typedef struct fid_tf {
    double t[3];
    double q[4];
} fid_tf;

/* add_fiducial service (addFiducialCallback, map.cpp:821-828): the next update that sees `fiducial_id` inserts it
 * (Map::handleAddFiducial, map.cpp:489-535, called by every Map::update at :173) as T_mapBase * T_baseCam * T_camFid with the
 * observation's variance, pins the origin fiducial's variance to 0 and ends map initialisation; a request for an id that is
 * already in the map is dropped.  T_mapBase = the host's tf lookup map -> base (map.cpp:514-517), NULL when it failed
 * ("Placing robot at the origin"). */
int fid_map_add_fiducial(fid_map* m, int instance, int fiducial_id, const fid_tf* T_mapBase);

typedef struct fid_robot_pose { /* geometry for /fiducial_pose (map.cpp:337-345) */
    int32_t valid;
    int32_t n_estimates;
    double t[3];
    double q[4];
    double variance;
} fid_robot_pose;

/* FiducialMapEntry (fiducial_msgs/msg/FiducialMapEntry.msg:2-10): x y z, roll pitch yaw (rad). */
typedef struct fid_map_entry {
    int32_t fiducial_id;
    int32_t num_obs;
    double x, y, z, rx, ry, rz;
    double variance;
} fid_map_entry;

/* One FiducialTransformArray message into one map instance.  Replaces
 * FiducialSlam::transformCallback (fiducial_slam/src/fiducial_slam.cpp:79-105) + Map::update
 * (fiducial_slam/src/map.cpp:152-176).  T_baseCam / T_camBase are the two tf lookups of
 * updatePose (map.cpp:258-273) performed by the host; NULL = that lookup failed. */
int fid_map_update(fid_map* m, int instance, int n_obs, const fid_transform* obs, const fid_tf* T_baseCam, const fid_tf* T_camBase, fid_robot_pose* robot);

/* A whole sequence of messages for every instance in one launch (bench config C5 / replay):
 * message k of instance i holds obs[offsets[i*(n_msgs+1)+k] .. offsets[i*(n_msgs+1)+k+1]).  robot
 * (optional) receives n_instances*n_msgs poses. */
int fid_map_update_sequence(fid_map* m, int n_msgs, const int32_t* offsets, const fid_transform* obs, const fid_tf* T_baseCam, const fid_tf* T_camBase,
                            fid_robot_pose* robot);

/* Same, fed straight from the dense output of fid_detect_pose_batch: frame f contributes
 * counts[f] transforms starting at transforms[f * max_markers]; one message per frame, in order, into
 * one instance (one camera stream). */
int fid_map_update_frames(fid_map* m, int instance, int n_frames, const int32_t* counts, const fid_transform* transforms, int max_markers, const fid_tf* T_baseCam,
                          const fid_tf* T_camBase, fid_robot_pose* last_robot);
/* Asynchronous form: the observations are copied and the update is enqueued on the map's stream; the
 * call returns at once so that the (sequential, latency-bound) fold overlaps the detection of the next
 * frames.  Every other fid_map_* call, and fid_map_sync, waits for pending updates first. */
int fid_map_update_frames_async(fid_map* m, int instance, int n_frames, const int32_t* counts, const fid_transform* transforms, int max_markers, const fid_tf* T_baseCam,
                                const fid_tf* T_camBase);
int fid_map_sync(fid_map* m);

/* publishMap (map.cpp:629-654): entries in ascending fiducial id. */
int fid_map_entries(fid_map* m, int instance, int max_entries, int* n, fid_map_entry* entries);

/* Batch SE(3) Gauss-Newton refinement of a map instance over a recorded message sequence (NEW -- SURVEY 8f-3, the north-star's
 * "batched SE(3) Gauss-Newton"; the reference only has the sequential fold above and the co-visibility links of map.cpp:217-222;
 * parity unpinned, stated and checked by oracle/refine_oracle.py, quality metric = fiducial_slam/scripts/fit_plane.py).
 * Unknowns: the instance's fiducial poses, entries with variance 0 stay fixed.  Every message that observes mapped fiducials a, b
 * (a before b) contributes the relative pose T_camFid_a^-1 T_camFid_b with weight 1 / (object_error_a + object_error_b + 1e-9);
 * cost = sum w (|Log(Z_R^T R_a^T R_b)|^2 + translation_weight |R_a^T (t_b - t_a) - Z_t|^2).  The poses are updated in place
 * (variances and observation counts are left alone).  Messages: obs[offsets[k] .. offsets[k+1]). */
typedef struct fid_refine_params {
    int32_t max_iterations;    /* Gauss-Newton steps, 1..64 (default 8) */
    int32_t pcg_iterations;    /* preconditioned conjugate-gradient iterations per step, upper bound (default 100) */
    double pcg_tolerance;      /* relative residual at which the linear solve stops (default 1e-10) */
    double damping;            /* Levenberg term on the diagonal (default 1e-6) */
    double translation_weight; /* lambda_t (default 1) */
} fid_refine_params;
typedef struct fid_refine_stats {
    double initial_cost, final_cost;
    double solve_ms; /* device time of the solve kernel (CUDA events on the map's stream) */
    int32_t iterations, n_edges, n_free, kernel_launches;
} fid_refine_stats;
int fid_map_refine_default_params(fid_refine_params* p);
int fid_map_refine(fid_map* m, int instance, int n_msgs, const int32_t* offsets, const fid_transform* obs, const fid_refine_params* params /* NULL = defaults */,
                   fid_refine_stats* stats /* optional */);

/* Multi-GPU merged map (NEW, no reference counterpart -- SURVEY 8e; parity unpinned, checked against
 * oracle/slam_oracle.py::merge_maps).  Every rank keeps its own LOCAL map instances (the reference's
 * sequential fold over its own camera stream).  Once per merge epoch each rank exports its instance as a
 * fixed-size table (max_fiducials records, ids ascending, unused records -1 at the end), the tables are
 * exchanged with ONE all-gather (ncclAllGather / torch.distributed.all_gather_into_tensor), and every
 * rank folds the gathered tables -- ranks in order, TransformWithVariance::update
 * (transform_with_variance.cpp:43-78), variance-0 entries win -- into a MERGED VIEW that is separate from
 * the local instances and rebuilt from scratch by every merge: merging is idempotent and nothing that was
 * exchanged at one epoch is fused again at the next. */
typedef struct fid_map_record {
    int32_t fiducial_id; /* -1 = empty slot */
    int32_t num_obs;
    double t[3];
    double q[4];
    double variance;
} fid_map_record;
int fid_map_export(fid_map* m, int instance, fid_map_record* table /* [max_fiducials] */);
/* Device pointer + byte size of the instance's export table (synchronous). */
int fid_map_export_device(fid_map* m, int instance, void** device_table, size_t* bytes);
/* Stream-ordered forms for an exchange that never blocks the host: fid_map_stream returns the
 * cudaStream_t every asynchronous fid_map_* call is ordered on; enqueue the export into a caller-owned
 * device buffer, the all-gather on that same stream, then the merge of the gathered buffer. */
int fid_map_stream(fid_map* m, void** cuda_stream);
int fid_map_export_async(fid_map* m, int instance, void* device_dst /* [max_fiducials] fid_map_record */);
int fid_map_merge_device_async(fid_map* m, int n_tables, const void* device_tables /* [n_tables][max_fiducials] */);
int fid_map_merge_device(fid_map* m, int n_tables, const void* device_tables);
int fid_map_merge(fid_map* m, int n_tables, const fid_map_record* tables /* host, [n_tables][max_fiducials] */);
/* The merged view as FiducialMapEntry fields (ids ascending), like fid_map_entries. */
int fid_map_merged_entries(fid_map* m, int max_entries, int* n, fid_map_entry* entries);
/* Replace an instance's fiducials by the merged view (explicit; its links are cleared). */
int fid_map_adopt_merged(fid_map* m, int instance);

/* ------------------------------------------------------------------------------------------------
 * JPEG ingest (NEW; SURVEY 8f-1).  Replaces the cv::imdecode that compressed_image_transport runs in front of
 * FiducialsNode::imageCallback (aruco_detect.cpp:332,348; default transport `compressed`,
 * aruco_detect/launch/aruco_detect.launch:6,28).  The Huffman bit stream of every image is decoded on host threads
 * (one image per thread); the sparse quantised coefficients (typically 4-6x smaller than the frame) cross PCIe and the
 * device performs dequantisation, the integer inverse DCT, chroma upsampling and the colour conversion, writing BGR8
 * frames into `device_bgr` -- the buffer fid_submit_batch / fid_detect_pose_batch take with bgr_on_device = 1.
 * Bit-exact against cv2.imdecode (libjpeg-turbo defaults).  Supported: baseline / extended-sequential 8-bit Huffman JPEG,
 * grey or YCbCr 4:4:4 / 4:2:2 / 4:2:0, restart intervals; other streams get status FID_ERR_UNSUPPORTED (decode those with
 * the host library and upload them as frames).  No CPU fallback: fid_jpeg_create fails with FID_ERR_NO_DEVICE.
 * ---------------------------------------------------------------------------------------------- */
typedef struct fid_jpeg fid_jpeg;
int fid_jpeg_create(int device, int max_width, int max_height, int max_batch, int n_threads /* 0 = one per hardware thread, at most 64 */, fid_jpeg** out);
int fid_jpeg_destroy(fid_jpeg* j);
/* n images, all width x height and of one sampling layout.  status[i] (optional) = FID_OK or the reason image i was skipped (its
 * frame is left untouched).  Returns once the device work is ENQUEUED on the decoder's stream (fid_jpeg_stream); fid_jpeg_sync
 * waits for it.  The call itself returns an error only when no image of the batch could be decoded. */
int fid_jpeg_decode_batch(fid_jpeg* j, int n, const uint8_t* const* data, const size_t* bytes, int width, int height, void* device_bgr, size_t row_stride,
                          size_t frame_stride, int32_t* status);
int fid_jpeg_sync(fid_jpeg* j);
int fid_jpeg_stream(fid_jpeg* j, void** cuda_stream);
/* last batch: wall time of the host entropy decoding, bytes copied to the device, device time (copies + kernels) */
int fid_jpeg_last_stats(fid_jpeg* j, double* host_decode_ms, double* h2d_bytes, double* device_ms);

#ifdef __cplusplus
}
#endif
#endif /* FIDUCIALS_B200_H */
