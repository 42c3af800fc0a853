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
 * marker order -- exactly what imageCallback copies into fiducial_msgs/Fiducial (:358-377).
 * Per-frame capacities (dense calibration targets reach them; DESIGN.md section 3): 4096 raw quad candidates (the quads of every
 * threshold window before grouping), 512 selected candidates (after grouping) and FID_MAX_MARKERS markers.  Past any of them the call
 * returns FID_ERR_CAPACITY and still writes *n and ids / corners[0 .. n):
 *   - more than 256 markers (raw and selected within capacity): n = 256, cv2's first 256 markers in cv2's order, cv2's corners;
 *   - more than 512 selected: the markers among the first 512 selected candidates (descending perimeter), at most 256;
 *   - more than 4096 raw candidates: the markers found among 4096 of them, at most 256; which 4096 are kept varies from call to call.
 *     A frame can get there with fewer than 256 markers (252 markers filling a 3840 x 2160 frame give 4200 raw candidates); fewer
 *     threshold windows (adaptiveThreshWinSizeMax) reduce the count. */
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
 * and the copy is part of the call.  Results always land in host arrays.
 * The per-frame capacities of fid_detect apply to every frame.  The status covers the whole batch: FID_ERR_CAPACITY when any frame
 * went past one of them (or has more markers than max_markers), and every frame's counts, ids, corners and transforms are written all
 * the same, each frame as fid_detect describes it; frames within the capacities get exactly the rows they get alone.
 * fid_collect_batch returns the same status for its batch. */
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

/* Both planar pose solutions of a marker (NEW; the reference publishes only the cv::solvePnP(SOLVEPNP_ITERATIVE) pose of
 * aruco_detect.cpp:247, and so does fid_transform).  A square seen small, far away or nearly fronto-parallel fits two poses
 * almost equally well, and ITERATIVE may settle in either.  Each record restates cv::solvePnPGeneric(obj, corners, K, D, rvecs,
 * tvecs, false, SOLVEPNP_IPPE_SQUARE, noArray(), noArray(), rms) of OpenCV 4.13 (IPPE::PoseSolver::solveSquare) on the object
 * points of estimatePoseSingleMarkers (getSingleMarkerObjectPoints :151-161, fiducial_len and its overrides narrowed to float):
 * the two solutions in solvePnPGeneric's order (by the IPPE solver's own error in normalised coordinates), each with the
 * reprojection RMS solvePnPGeneric reports (projectPoints with K and D, norm / sqrt(2n), px).  iterative_match = index of the
 * solution whose rotation is closer to the ITERATIVE pose of the marker's fid_transform: 0 when the published pose is the
 * better-fitting hypothesis, 1 when it is the other one.  n = 0 (everything else 0, iterative_match -1) where solvePnPGeneric
 * finds no solution: a degenerate quad.  The published pose and every other output are unchanged.
 * A struct tag without a typedef: the plain name is the function fid_pose_hypotheses below, so write `struct fid_pose_hypotheses`. */
struct fid_pose_hypotheses {
    int32_t fiducial_id;
    int32_t n;                /* 2; 0 if IPPE found no solution (degenerate quad) */
    int32_t iterative_match;  /* which of the two the ITERATIVE pose of fid_transform lies in; -1 when n == 0 */
    int32_t reserved;
    double rvec[2][3], tvec[2][3];
    double rms[2];            /* reprojection RMS in px, in cv::solvePnPGeneric's order */
};

/* Opt-in second pose stage of the batch calls (default off): with it on, every batch submitted with a camera also computes the
 * records of its markers on the device, after the ITERATIVE pose, and copies them back with the other results.  Not while
 * batches are in flight (like fid_set_input_encoding).  The first enable allocates the result buffers. */
int fid_set_pose_hypotheses(fid_detector* h, int enable);
/* Records for markers already detected, the counterpart of fid_pose (same arguments, same object points and overrides); it runs
 * the ITERATIVE solve of fid_pose itself for iterative_match.  Works whether or not the batch option is on. */
int fid_pose_hypotheses(fid_detector* h, int n, const int32_t* ids, const float* corners, const fid_camera* cam, double fiducial_len, int n_override,
                        const int32_t* override_ids, const double* override_lens, struct fid_pose_hypotheses* out);
/* Records of the batch most recently returned by fid_collect_batch / fid_detect_pose_batch, dense [n_frames][max_markers] in
 * the marker order of that batch's ids and transforms (records past counts[f] are not written).  *n_frames = the batch's frame
 * count; out may be NULL to query it.  FID_ERR_INVALID_ARG if the option was off for that batch (or it had no camera);
 * FID_ERR_CAPACITY, with nothing written, if a frame of the batch has more markers than max_markers. */
int fid_last_pose_hypotheses(fid_detector* h, int max_markers, int* n_frames, struct fid_pose_hypotheses* out);

/* One pose per marker board (NEW; the reference publishes per-marker poses only -- fiducial_slam reads a
 * `multi_error_theshold` for a multi-fiducial pose, map.cpp:127-129, that it never computes).  A board is a known rigid layout of
 * markers (a docking station, a calibration target, tags on one plate); its pose restates what OpenCV 4.13 users compute with
 * cv::aruco::Board::matchImagePoints(corners, ids) + cv::solvePnP(SOLVEPNP_ITERATIVE, no extrinsic guess): every detection whose id
 * is on the board, in detection order, contributes that marker's 4 object points and its 4 corners (a repeated detection
 * contributes twice), and one solvePnP runs over all of them (planar or 3-D boards; the branch follows the matched points).
 * image_error is getReprojectionError (aruco_detect.cpp:203-221) over every matched point; rotation is packed as :447-448. */
#define FID_MAX_BOARDS 16
typedef struct fid_board {
    int32_t n_markers;          /* 1..4096, distinct ids */
    const int32_t* ids;         /* [n_markers] */
    const float* obj_points;    /* [n_markers][4][3], metres, marker corner order of cv::aruco::Board */
} fid_board;
typedef struct fid_board_pose {
    int32_t board;              /* index into the fid_set_boards array */
    int32_t status;             /* 1 pose, 0 no board marker detected, -1 non-planar and < 6 points (cv2 raises) */
    int32_t n_markers, n_points;
    double rvec[3], tvec[3], rotation[4];   /* rotation = quaternion x y z w */
    double image_error;         /* mean squared reprojection error, px^2 */
} fid_board_pose;
/* Set the boards of the handle (copied; 0 boards = off, the default).  With boards set, every batch submitted with a camera also
 * solves one pose per (frame, board) on the device, after the per-marker poses, and copies the records back with the other
 * results; without boards the batch calls launch exactly what they launch otherwise.  FID_ERR_INVALID_ARG for sizes out of range,
 * a non-finite object point, an id repeated within one board (a detection could not say which marker it is), or while batches
 * are in flight. */
int fid_set_boards(fid_detector* h, int n_boards, const fid_board* boards);
/* Board poses for markers already detected (0 <= n <= FID_MAX_MARKERS; ids / corners as fid_detect returns them), the counterpart
 * of fid_pose: out[n_boards] in board order.  FID_ERR_INVALID_ARG if no boards are set. */
int fid_estimate_board_poses(fid_detector* h, int n, const int32_t* ids, const float* corners, const fid_camera* cam, fid_board_pose* out);
/* Records of the batch most recently returned by fid_collect_batch / fid_detect_pose_batch, dense [n_frames][max_boards] in board
 * order.  *n_frames, *n_boards = that batch's counts; out may be NULL to query them.  FID_ERR_INVALID_ARG if that batch ran
 * without boards or without a camera; FID_ERR_CAPACITY, with nothing written, if max_boards < *n_boards. */
int fid_last_board_poses(fid_detector* h, int max_boards, int* n_frames, int* n_boards, fid_board_pose* out);

/* ChArUco boards (NEW): a chessboard with a marker in every white square, as cv::aruco::CharucoBoard(size, squareLength,
 * markerLength, dictionary, ids) of OpenCV 4.13 lays it out.  Its chessboard corners are found from the detected markers as
 * cv::aruco::CharucoDetector::detectBoard(image, charucoCorners, charucoIds, markerCorners, markerIds) finds them for markers it is
 * given (with a camera through an approximate solvePnP over the markers, without one through each marker's local homography;
 * cornerSubPix with per-corner windows of 1..10 px and the detector's cornerRefinementMaxIterations / MinAccuracy; minMarkers and
 * checkMarkers), and the board pose is CharucoBoard::matchImagePoints(corners, ids) + cv::solvePnP(SOLVEPNP_ITERATIVE). */
#define FID_MAX_CHARUCO_BOARDS 16
#define FID_MAX_CHARUCO_CORNERS 1024 /* per board: (squares_x - 1) (squares_y - 1) */
typedef struct fid_charuco_board {
    int32_t squares_x, squares_y;  /* >= 2 each */
    float square_length, marker_length;  /* metres, 0 < marker_length < square_length */
    int32_t legacy_pattern;        /* CharucoBoard::setLegacyPattern */
    const int32_t* ids;            /* [squares_x * squares_y / 2] distinct marker ids, or NULL for 0 .. n - 1 */
    int32_t min_markers;           /* CharucoParameters::minMarkers, 0..2 (cv2 default 2) */
    int32_t check_markers;         /* CharucoParameters::checkMarkers (cv2 default 1) */
} fid_charuco_board;
typedef struct fid_charuco_result {
    int32_t board;                 /* index into the fid_set_charuco_boards array */
    int32_t n_corners;             /* corners found */
    int32_t corner_offset;         /* first slot of this board in the per-frame corner arrays */
    int32_t status;                /* 1 pose, 0 no camera or < 4 corners, -2 collinear corners, -3 rejected by checkMarkers (the
                                      corners are coplanar, so solvePnP's -1 of fid_board_pose cannot occur) */
    double rvec[3], tvec[3], rotation[4];  /* rotation = quaternion x y z w */
    double image_error;            /* mean squared reprojection error of the corners, px^2 */
} fid_charuco_result;
/* Set the ChArUco boards of the handle (the layout is computed from these numbers; 0 boards = off, the default).  Each board owns
 * (squares_x - 1)(squares_y - 1) slots of the per-frame corner arrays, board after board; its n_corners first slots hold the
 * corners in ascending corner id (cv2's order), the others id -1 and (-1, -1).  With boards set, every batch also finds the corners
 * of each (frame, board) on the device after the other stages, with or without a camera (no pose without one), and copies them
 * back with the other results; without boards the batch calls launch exactly what they launch otherwise.  FID_ERR_INVALID_ARG for
 * sizes out of range, repeated ids within a board, more markers than the dictionary has, or while batches are in flight. */
int fid_set_charuco_boards(fid_detector* h, int n_boards, const fid_charuco_board* boards);
/* Corners and pose of every ChArUco board set, for one frame (in the fid_set_input_encoding format) and markers already detected
 * (0 <= n <= FID_MAX_MARKERS; ids / corners as fid_detect returns them): the counterpart of detectBoard(image, markerCorners,
 * markerIds).  cam may be NULL.  results[n_boards]; corner_ids / corner_xy [total slots] ([2] floats per slot).  No marker: no
 * corner.  FID_ERR_INVALID_ARG if no boards are set or while batches are in flight. */
int fid_detect_charuco(fid_detector* h, const uint8_t* bgr, int width, int height, size_t stride, int n, const int32_t* ids, const float* corners,
                       const fid_camera* cam, fid_charuco_result* results, int32_t* corner_ids, float* corner_xy);
/* Records and corners of the batch most recently returned by fid_collect_batch / fid_detect_pose_batch: results dense
 * [n_frames][n_boards], corners dense [n_frames][max_slots].  *n_frames, *n_boards, *n_slots = that batch's counts; results may
 * be NULL to query them.  FID_ERR_INVALID_ARG if that batch ran without ChArUco boards; FID_ERR_CAPACITY, with nothing written, if
 * max_slots < *n_slots. */
int fid_last_charuco(fid_detector* h, int max_slots, int* n_frames, int* n_boards, int* n_slots, fid_charuco_result* results, int32_t* corner_ids,
                     float* corner_xy);

/* Recovery of missed board markers (NEW), as cv::aruco::ArucoDetector::refineDetectedMarkers(image, board, detectedCorners,
 * detectedIds, rejectedCorners, K, D, recoveredIdxs) of OpenCV 4.13 computes it with RefineParameters(min_rep_distance,
 * error_correction_rate, check_all_orders).  The board predicts where each of its markers that was not detected should be (with a
 * camera through solvePnP over the detected board markers and projectPoints; without one through a homography, for boards whose points
 * share one z); the first rejected candidate, in list order, whose corners all lie within min_rep_distance of the prediction and whose
 * inner bits differ from the marker's code in fewer than int(max correction bits * error_correction_rate) bits (no bit check when
 * error_correction_rate < 0) becomes that marker, with cornerSubPix under CORNER_REFINE_SUBPIX.  Every marker board set with
 * fid_set_boards, then every ChArUco board set with fid_set_charuco_boards, is one such call on the lists the previous call left. */
#define FID_MAX_REJECTED 4096
typedef struct fid_marker_refine_params {
    int32_t enable;                /* 0 = off (the default) */
    float min_rep_distance;        /* px, > 0 (cv2 default 10) */
    float error_correction_rate;   /* cv2 default 3; < 0 = no bit check; 0 recovers nothing (the bit test is strict) */
    int32_t check_all_orders;      /* try the 4 corner orders of a candidate (cv2 default 1) */
} fid_marker_refine_params;
/* Set the refinement parameters (copied).  fid_refine_detected_markers uses them, and so do the batch calls once
 * fid_set_batch_marker_refinement is on; this call alone changes nothing in the batch calls.  FID_ERR_INVALID_ARG for
 * min_rep_distance <= 0 or non-finite values, or while batches are in flight. */
int fid_set_marker_refinement(fid_detector* h, const fid_marker_refine_params* params);
/* Refinement inside the batch calls (fid_detect_pose_batch, fid_submit_batch; 0 = off, the default).  A batch refines when this
 * switch is on, fid_set_marker_refinement is enabled and at least one marker or ChArUco board is set; otherwise it launches exactly
 * what it launches without the switch.  A refining batch recovers, per frame, the missed board markers from its own rejected list
 * (fid_debug_rejected's rule) after detection and before the board pose and ChArUco stages, which then see the recovered markers.
 * Detected markers keep their slots, corners and poses; recovered markers are appended after them in recovery order, with a pose
 * when the batch has a camera, and counts include them.  When a recovered marker finds no slot below max_markers, the frame stops
 * refining there and the batch returns FID_ERR_CAPACITY.  fid_detect never refines.  The first enable allocates the buffers.
 * FID_ERR_INVALID_ARG while batches are in flight. */
int fid_set_batch_marker_refinement(fid_detector* h, int enable);
/* The refinement of the batch most recently returned by fid_collect_batch / fid_detect_pose_batch: per frame n_recovered[f],
 * recovered_idx / recovered_board [f][max_markers] (as fid_refine_detected_markers reports them; the recovered markers are the last
 * n_recovered[f] of the frame's markers), n_rejected[f] and rejected [f][max_rejected][4][2]: the frame's rejected list BEFORE
 * refinement, which recovered_idx indexes.  Output pointers may be NULL.  FID_ERR_INVALID_ARG if that batch did not refine;
 * FID_ERR_CAPACITY, with nothing written, if a frame has more recovered markers than max_markers or more rejected candidates than
 * max_rejected (for the arrays passed). */
int fid_last_marker_refinement(fid_detector* h, int max_markers, int max_rejected, int* n_frames, int32_t* n_recovered, int32_t* recovered_idx,
                               int32_t* recovered_board, int32_t* n_rejected, float* rejected);
/* refineDetectedMarkers for one frame (in the fid_set_input_encoding format) and lists the caller already has, against every board
 * set: ids / corners hold n detections ([.][4][2] floats) and receive the recovered markers after them (capacity max_markers <=
 * FID_MAX_MARKERS); rejected [n_rejected][4][2] (n_rejected <= FID_MAX_REJECTED) is detectMarkers' rejectedImgPoints.  cam may be
 * NULL.  *n_out = the number of detections after; recovered_idx / recovered_board [max_markers]: per recovered marker, in recovery
 * order, its index into rejected as passed in and its board (b for marker board b, FID_MAX_BOARDS + c for ChArUco board c).
 * FID_ERR_INVALID_ARG if refinement is off, no board is set or while batches are in flight; FID_ERR_CAPACITY, with nothing written,
 * if the recovered markers do not fit in max_markers. */
int fid_refine_detected_markers(fid_detector* h, const uint8_t* bgr, int width, int height, size_t stride, int n, int32_t* ids, float* corners,
                                int max_markers, int n_rejected, const float* rejected, const fid_camera* cam, int* n_out, int32_t* recovered_idx,
                                int32_t* recovered_board);

/* ChArUco diamonds (NEW): a 3x3 chessboard with four markers around the centre square, named by the four marker ids, as
 * cv::aruco::CharucoDetector(CharucoBoard((3, 3), square_length, marker_length, dictionary)).detectDiamonds(image, diamondCorners,
 * diamondIds, markerCorners, markerIds) of OpenCV 4.13 finds them among markers it is given.  Each marker in list order that is not
 * part of a diamond yet tries to become the top marker of one: refineDetectedMarkers against a temporary diamond with the ids
 * {id, id + 2, id + 3, id + 4} and no camera looks for the other three among the remaining markers (within 1.302455 times the root
 * of the sum of the marker's squared sides; with CORNER_REFINE_SUBPIX the markers it takes get cornerSubPix, and cv2 keeps that
 * change in its marker list, as this library does internally); when all three are found, detectBoard on the temporary board (the
 * detector's camera if set, otherwise local homographies; min_markers, check_markers) gives the four chessboard corners.  A diamond
 * is reported when all four survive, in the order found, its corners in cv2's order (0, 1, 3, 2 of the board's corner ids).  With a
 * camera its pose is cv::solvePnP(SOLVEPNP_ITERATIVE) of the corners on getSingleMarkerObjectPoints(square_length), packed as every
 * fid_transform (fid_pose's arithmetic, square_length as the marker length). */
#define FID_MAX_DIAMONDS (FID_MAX_MARKERS / 4) /* per frame: every diamond takes four markers */
typedef struct fid_diamond_params {
    int32_t enable;                /* 0 = off (the default) */
    float square_length, marker_length;  /* metres, 0 < marker_length < square_length */
    int32_t min_markers;           /* CharucoParameters::minMarkers, 0..2 (cv2 default 2) */
    int32_t check_markers;         /* CharucoParameters::checkMarkers (cv2 default 1) */
} fid_diamond_params;
typedef struct fid_diamond {
    int32_t ids[4];                /* cv2's diamondIds: the top marker, then the ones found at the left, right and bottom */
    float corners[8];              /* x0, y0 .. x3, y3 */
    int32_t status;                /* 1 pose, 0 no camera */
    fid_transform pose;            /* fiducial_id = ids[0] */
} fid_diamond;
/* Set the diamond geometry of the handle (one per handle, as one cv2 CharucoDetector; copied).  With it on, every batch
 * (fid_detect_pose_batch, fid_submit_batch) also finds the diamonds of each frame on the device after every other stage, from the
 * frame's final markers (those recovered by batch refinement included), with the batch's camera; without a camera there is no pose.
 * fid_detect stays detectMarkers alone.  With it off the batch calls launch exactly what they launch otherwise.  The first enable
 * allocates the buffers.  FID_ERR_INVALID_ARG for non-finite or out-of-range values, or while batches are in flight. */
int fid_set_diamonds(fid_detector* h, const fid_diamond_params* params);
/* The diamonds of one frame (in the fid_set_input_encoding format) and markers already detected (0 <= n <= FID_MAX_MARKERS; ids /
 * corners as fid_detect returns them; they are not changed): *n_diamonds records in out, which has room for n / 4.  cam may be
 * NULL.  FID_ERR_INVALID_ARG if diamonds are off or while batches are in flight. */
int fid_detect_diamonds(fid_detector* h, const uint8_t* bgr, int width, int height, size_t stride, int n, const int32_t* ids, const float* corners,
                        const fid_camera* cam, int* n_diamonds, fid_diamond* out);
/* The diamonds of the batch most recently returned by fid_collect_batch / fid_detect_pose_batch: counts[f] and out dense
 * [n_frames][max_diamonds].  *n_frames = that batch's frame count; counts and out may be NULL to query it.  FID_ERR_INVALID_ARG if
 * that batch ran without diamonds; FID_ERR_CAPACITY, with nothing written, if a frame has more than max_diamonds. */
int fid_last_diamonds(fid_detector* h, int max_diamonds, int* n_frames, int32_t* counts, fid_diamond* out);

/* Several dictionaries in one pass: cv::aruco::ArucoDetector(dictionaries) and detectMarkersMultiDict (OpenCV >= 4.12).  The
 * threshold, border walk and quad stages run once per frame; grouping runs once per run of equal marker sizes, and identification,
 * the candidate hierarchy, corner refinement and the pose once per dictionary.  The markers are the concatenation, in list order,
 * of what detectMarkers returns for each dictionary alone (a dictionary listed twice reports its markers twice).
 *   dictionary    the OpenCV enum (the fid_params.dictionary values)
 *   id_offset     fid_transform.fiducial_id = id + id_offset ("published id"), so that two families with equal raw ids stay apart
 *                 in the map; ids and corners stay cv2's raw values
 *   fiducial_len  metres, 0 = the call's fiducial_len.  A marker's length is the fiducial_len_override entry of its published id,
 *                 else this length if > 0, else the call's; object_error uses this length (else the call's) as the default length. */
#define FID_MAX_DICTIONARIES 8
typedef struct fid_dictionary_spec {
    int32_t dictionary;
    int32_t id_offset;
    double fiducial_len;
} fid_dictionary_spec;
/* Replace the handle's dictionary list (1..FID_MAX_DICTIONARIES entries); entry 0's dictionary becomes fid_params.dictionary, and
 * fid_set_params later replaces entry 0's dictionary and keeps the others (cv2's setDictionary).  Every entry must pass the limits
 * fid_create applies to fid_params.dictionary: FID_ERR_UNSUPPORTED / FID_ERR_INVALID_ARG otherwise, also for a length that is
 * negative or not finite or an offset with which id + id_offset overflows int32, each with the handle unchanged.  A handle is in
 * multi-dictionary mode when the list has more than one entry or entry 0 has an offset or a length; the batch calls then detect
 * with every dictionary.  Batch marker refinement, and boards, ChArUco boards and diamonds set without a family (fid_set_boards,
 * fid_set_charuco_boards, fid_set_diamonds), are refused (FID_ERR_UNSUPPORTED, nothing changed) in that mode, in both directions.
 * With boards bound to families (fid_set_family_*), a new list is accepted when every bound index still names an entry of it;
 * FID_ERR_INVALID_ARG, with the handle unchanged, when a bound index would not, or when a bound ChArUco board has more markers than
 * its new family's dictionary.  Not while batches are in flight. */
int fid_set_dictionaries(fid_detector* h, int n, const fid_dictionary_spec* specs);
/* Boards bound to dictionary families (NEW): fid_set_boards, fid_set_charuco_boards and fid_set_diamonds, each board (or the
 * diamonds) bound to an entry of the handle's dictionary list, dict_index in fid_set_dictionaries order.  Raw ids repeat across
 * families (DICT_4X4_50 id 3 and DICT_5X5_1000 id 3 are different markers), so in multi-dictionary mode a stage bound to family k
 * reads that family's markers alone, in list order: what a cv2 4.13 user gets by running Board::matchImagePoints + solvePnP,
 * CharucoDetector(CharucoBoard(..., dicts[k], ids)).detectBoard and CharucoDetector(CharucoBoard((3, 3), ..., dicts[k]))
 * .detectDiamonds on corners[di == k], ids[di == k] of detectMarkersMultiDict, with family k's detector parameters.  A diamond's
 * pose.fiducial_id is ids[0] + family k's id_offset (its ids stay raw).  The batch calls (fid_detect_pose_batch, fid_submit_batch /
 * fid_collect_batch) run the stages after the merge and fid_last_board_poses / fid_last_charuco / fid_last_diamonds return them as
 * usual; fid_detect_multi_dict runs the ChArUco stage as fid_detect does.  fid_estimate_board_poses, fid_detect_charuco,
 * fid_detect_diamonds and fid_refine_detected_markers return FID_ERR_UNSUPPORTED in multi-dictionary mode (their lists carry no
 * family), and fid_detect there runs no board stage.  Each call accepts what its counterpart accepts, plus
 * 0 <= dict_index < the number of entries (FID_ERR_INVALID_ARG, handle unchanged, otherwise); on a single-dictionary handle index 0
 * gives exactly the counterpart's outputs. */
int fid_set_family_boards(fid_detector* h, int n_boards, const fid_board* boards, const int32_t* dict_index);
int fid_set_family_charuco_boards(fid_detector* h, int n_boards, const fid_charuco_board* boards, const int32_t* dict_index);
int fid_set_family_diamonds(fid_detector* h, const fid_diamond_params* params, int32_t dict_index);
/* detectMarkersMultiDict for one frame (fid_detect's arguments): ids, corners and dict_indices (may be NULL) [n], max_markers a
 * total over all dictionaries (FID_ERR_CAPACITY with the first max_markers written beyond it).  fid_detect stays detectMarkers
 * with dictionary 0 alone, as cv2's detectMarkers on a detector with several dictionaries. */
int fid_detect_multi_dict(fid_detector* h, const uint8_t* bgr, int width, int height, size_t stride, int max_markers, int* n, int32_t* ids, float* corners,
                          int32_t* dict_indices);
/* The dictionary index of every marker of the batch most recently returned by fid_collect_batch / fid_detect_pose_batch, dense
 * [n_frames][max_markers] (all zeros without multi-dictionary mode).  *n_frames = that batch's frame count; out may be NULL to query
 * it.  FID_ERR_INVALID_ARG before the first batch; FID_ERR_CAPACITY, with nothing written, if a frame has more than max_markers. */
int fid_last_dict_indices(fid_detector* h, int max_markers, int* n_frames, int32_t* out);

/* Detection on a downscaled frame with pyramid corner upsampling: DetectorParameters.useAruco3Detection of OpenCV 4.13
 * (Romero-Ramirez et al. 2018).  Off by default.  With enable set, fid_detect, fid_detect_pose_batch and fid_submit_batch /
 * fid_collect_batch return what cv2.aruco.ArucoDetector(dictionary, params).detectMarkers returns with useAruco3Detection = True,
 * minSideLengthCanonicalImg and minMarkerLengthRatioOriginalImg as given:
 *   - the threshold, border-walk, quad and grouping stages run on the gray frame resized (INTER_LINEAR) by
 *     fxfy = minSide / (minSide + max(W, H) * ratio), with a minimum contour length of 4 * minSide in place of
 *     minMarkerPerimeterRate;
 *   - each candidate's bits are read from the level of the frame's pyrDown pyramid that its contour length picks;
 *   - the corners are brought back to full resolution by cornerSubPix on the pyramid levels (windows 3 and 5), whatever
 *     cornerRefinementMethod says; with ratio 0 the frame is not scaled and no cornerSubPix runs.
 * The pose and everything after it (pose hypotheses, boards, ChArUco, diamonds) receive the full-resolution corners and frame.
 * Refused (FID_ERR_UNSUPPORTED, nothing changed), in both directions: several dictionaries (fid_set_dictionaries with a list that
 * makes the handle multi-dictionary, fid_detect_multi_dict) and batch marker refinement; fid_debug_rejected refuses while the mode
 * is on.  minSideLengthCanonicalImg 1..16384, minMarkerLengthRatioOriginalImg 0..1 (FID_ERR_INVALID_ARG otherwise).  An enable
 * allocates each slot's pyramid and segmentation planes at the size its parameters need for frames up to fid_create's maximum (the
 * segmentation plane is never larger than the frame, and not allocated at ratio 0), and grows them when later parameters need more.
 * Not while batches are in flight. */
typedef struct fid_aruco3_params {
    int32_t enable;
    int32_t minSideLengthCanonicalImg;       /* cv2 default 32 */
    double minMarkerLengthRatioOriginalImg;  /* cv2 default 0 */
} fid_aruco3_params;
int fid_set_aruco3(fid_detector* h, const fid_aruco3_params* params);
/* The planes the mode builds for one frame (fid_detect's arguments), for locating a mismatch: info[4] = segmentation width,
 * height, pyramid levels (level 0 included) and the level the corners start from; seg [seg_h][seg_w] (may be NULL); pyramid: levels
 * 1 .. n - 1 concatenated, each [h][w] with w = (w_above + 1) / 2 (may be NULL; level 0 is the gray plane of fid_debug_threshold).
 * pyramid_bytes = the capacity of `pyramid` (FID_ERR_CAPACITY if it is too small).  With seg and pyramid both NULL only info is
 * filled, without device work.  FID_ERR_INVALID_ARG while the mode is off. */
int fid_debug_aruco3_planes(fid_detector* h, const uint8_t* bgr, int width, int height, size_t stride, int32_t* info, uint8_t* seg, uint8_t* pyramid,
                            size_t pyramid_bytes);

/* Per-marker detection confidence: cv2.aruco.ArucoDetector.detectMarkersWithConfidence of OpenCV 4.13.  A marker's confidence is
 * 1 - the mean over its cells of the share of each cell's sampling window that disagrees with the decoded marker (black border,
 * the dictionary word of the id inside), on the canonical image identification reads: 1.0 for a clean marker, lower for cells
 * that error correction fixed, partial occlusion or glare.  float32, computed at identification (whatever
 * cornerRefinementMethod says; on the pyramid level with useAruco3Detection).
 * fid_detect_with_confidence: one frame (fid_detect's arguments); ids and corners exactly as fid_detect returns them, and
 * confidence[n] (may be NULL).  Works whether or not the batch option is on.  FID_ERR_UNSUPPORTED in multi-dictionary mode (cv2
 * has no confidence for detectMarkersMultiDict). */
int fid_detect_with_confidence(fid_detector* h, const uint8_t* bgr, int width, int height, size_t stride, int max_markers, int* n, int32_t* ids, float* corners,
                               float* confidence);
/* Opt-in confidence of the batch calls (default off): with it on, fid_detect_pose_batch and fid_submit_batch / fid_collect_batch
 * also compute every marker's confidence; ids, corners and transforms are unchanged.  Refused (FID_ERR_UNSUPPORTED, nothing
 * changed), in both directions: several dictionaries (fid_set_dictionaries) and batch marker refinement (recovered markers have no
 * cv2 confidence).  Not while batches are in flight.  The first use allocates the result buffers. */
int fid_set_marker_confidence(fid_detector* h, int enable);
/* Confidences of the batch most recently returned by fid_collect_batch / fid_detect_pose_batch (or fid_detect_with_confidence),
 * dense [n_frames][max_markers] in the marker order of that batch (entries past counts[f] are not written).  *n_frames = the
 * batch's frame count; out may be NULL to query it.  FID_ERR_INVALID_ARG if the option was off for that batch; FID_ERR_CAPACITY,
 * with nothing written, if a frame of the batch has more markers than max_markers. */
int fid_last_marker_confidence(fid_detector* h, int max_markers, int* n_frames, float* out);

/* detectInvertedMarker of OpenCV 4.13 (default off): also detect white-on-black markers (engraved or laser-etched plates, markers
 * on dark surfaces, screens).  Every candidate's border is checked in both polarities and read in the one with fewer border errors
 * (a tie keeps black-on-white); its confidence is measured against that polarity.  As in cv2, the flag also changes which outline
 * of a group of nested candidates is kept: the smallest instead of the largest, so ordinary black markers come back with other
 * corners and possibly in another order.  Applies to fid_detect, fid_detect_pose_batch, fid_submit_batch / fid_collect_batch,
 * fid_detect_multi_dict, fid_detect_with_confidence and useAruco3Detection.  Refused (FID_ERR_UNSUPPORTED, nothing changed), in
 * both directions: batch marker refinement and marker refinement (fid_set_batch_marker_refinement, fid_set_marker_refinement,
 * fid_refine_detected_markers); fid_debug_rejected refuses while the flag is on.  Not while batches are in flight. */
int fid_set_detect_inverted_marker(fid_detector* h, int enable);

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
/* detectMarkers' rejectedImgPoints for the last fid_detect call on slot 0: the selected candidates that are not markers (not
 * decoded, or never reached by OpenCV 4.13's candidate hierarchy), in selection order (descending perimeter), each with its own
 * integer corners in the clockwise order of the candidate stage, neither rotated nor refined.  rejected [n][4][2] floats (may be
 * NULL).  *n = the count; FID_ERR_CAPACITY if it exceeds max_rejected; FID_ERR_INVALID_ARG before the handle's first fid_detect. */
int fid_debug_rejected(fid_detector* h, int max_rejected, int* n, float* rejected);

/* Per-stage device times (milliseconds, CUDA events) of the last batch call:
 * [0] h2d copy, [1] threshold (+ start cracks), [2] unused (reads 0), [3] border walk, [4] chain emit, [5] polygon+filters,
 * [6] group, [7] identify, [8] subpix+pose, [9] unused, [10] d2h, [11..18] the border-walk rounds
 * (unused rounds read 0); n_stages returns 19.  In multi-dictionary mode (fid_set_dictionaries) the per-dictionary launches interleave:
 * [6] then holds grouping, identification and the output stage of every dictionary, [7] reads 0 and [8] is the merge (k_dict_merge). */
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
 * Camera calibration.  Replaces cv::calibrateCameraExtended (OpenCV 4.13, calib3d/src/calibration.cpp) for the camera model of
 * fid_camera (K and k1 k2 p1 p2 k3): the initial intrinsics of cvInitIntrinsicParams2D (planar rigs) or the caller's guess, one
 * findExtrinsicCameraParams2 per view, then the joint Levenberg-Marquardt of cv2's CvLevMarq schedule, every view's step solved
 * on the device through the Schur complement of the 9 intrinsics.  Standalone: no detector handle; the device buffers and the
 * stream are the call's own and are released before it returns.
 * ---------------------------------------------------------------------------------------------- */
#define FID_CALIB_USE_INTRINSIC_GUESS 0x00001 /* the flag values are cv2's CALIB_* */
#define FID_CALIB_FIX_ASPECT_RATIO 0x00002
#define FID_CALIB_FIX_PRINCIPAL_POINT 0x00004
#define FID_CALIB_ZERO_TANGENT_DIST 0x00008
#define FID_CALIB_FIX_FOCAL_LENGTH 0x00010
#define FID_CALIB_FIX_K1 0x00020
#define FID_CALIB_FIX_K2 0x00040
#define FID_CALIB_FIX_K3 0x00080
#define FID_CALIB_MAX_VIEWS 65536
#define FID_CALIB_MAX_POINTS 4096       /* per view */
#define FID_CALIB_MAX_TOTAL (1 << 24)   /* points over all views */
#define FID_CALIB_MAX_STEPS 2048        /* recorded trial steps (a run takes at most 2 max_iter + 20) */
/* fid_calib_result.status: why the call returned FID_ERR_INVALID_ARG where cv2 raises */
#define FID_CALIB_OK 0
#define FID_CALIB_E_POINTS 1     /* a view with fewer than 4 points (or more than FID_CALIB_MAX_POINTS) */
#define FID_CALIB_E_NONPLANAR 2  /* no intrinsic guess and an object z off 0 (mean or standard deviation above 1e-5) */
#define FID_CALIB_E_HOMOGRAPHY 3 /* initIntrinsicParams2D: a view's points give no homography (e.g. collinear) */
#define FID_CALIB_E_GUESS 4      /* the guess: fx, fy <= 0, principal point outside the image, or an aspect ratio outside [0.01, 100] */
#define FID_CALIB_E_EXTRINSICS 5 /* findExtrinsicCameraParams2 raises: non-planar view with fewer than 6 points, degenerate DLT */
#define FID_CALIB_E_INPUT 6      /* non-finite points, bad offsets or sizes */
#define FID_CALIB_E_RO_VIEWS 7   /* fid_calibrate_camera_ro releasing: views of different sizes or with different object points */
#define FID_CALIB_E_RO_SINGULAR 8 /* fid_calibrate_camera_ro releasing: a non-positive pivot in the reduced system (DESIGN.md finding 21) */
#define FID_CALIB_E_RO_RESIDUALS 9 /* fid_calibrate_camera_ro releasing: as many free parameters as residuals (2 per point) or more */
/* cv::TermCriteria: type bit 1 = COUNT (max_iter, clamped to 1..1000; else 30), bit 2 = EPS (epsilon; else DBL_EPSILON) */
typedef struct fid_calib_criteria {
    int32_t type;
    int32_t max_iter;
    double epsilon;
} fid_calib_criteria;
typedef struct fid_calib_result {
    double rms;                   /* cv2's return value */
    fid_camera camera;            /* cameraMatrix, distCoeffs */
    double std_intrinsics[9];     /* stdDeviationsIntrinsics[0..8] = fx fy cx cy k1 k2 p1 p2 k3 (cv2's entries 9..17 are 0) */
    int32_t iterations;           /* CvLevMarq iterations */
    int32_t status;               /* FID_CALIB_* */
} fid_calib_result;
typedef struct fid_calib_stats {
    int32_t n_steps;              /* trial steps taken */
    int32_t n_evaluations;        /* Jacobian evaluations (the final one for the standard deviations included) */
    int32_t kernel_launches;
    int32_t reserved;
    double device_ms;             /* CUDA events around the device work */
    uint8_t steps[FID_CALIB_MAX_STEPS]; /* per trial step: 1 kept, 0 rejected (raised lambda) */
} fid_calib_stats;
/* n_views views, view v = points offsets[v] .. offsets[v+1] (offsets[0] = 0) of obj [.][3] and img [.][2] (float32, host).  guess:
 * K and D for FID_CALIB_USE_INTRINSIC_GUESS, and the aspect ratio K[0] / K[4] for FID_CALIB_FIX_ASPECT_RATIO (NULL = identity K,
 * zero D).  criteria NULL = cv2's default (COUNT + EPS, 30, DBL_EPSILON).  Outputs (host, optional but result): rvecs, tvecs
 * [n_views][3], std_extrinsics [n_views][6] (rvec then tvec), per_view_errors [n_views].  FID_ERR_UNSUPPORTED for any other
 * flag (rational, thin-prism, tilted models, FIX_K4 and up, ...); FID_ERR_INVALID_ARG with result->status where cv2 raises or the
 * caps above are exceeded; FID_ERR_NO_DEVICE without a usable device. */
int fid_calibrate_camera(int device, int n_views, const int32_t* offsets, const float* obj, const float* img, int width, int height, const fid_camera* guess,
                         int32_t flags, const fid_calib_criteria* criteria, fid_calib_result* result, double* rvecs, double* tvecs, double* std_extrinsics,
                         double* per_view_errors, fid_calib_stats* stats /* optional */);

/* cv::calibrateCameraROExtended: fid_calibrate_camera's calibration that also re-estimates the object points (the object-releasing
 * method of Strobl and Hirzinger), for boards whose printed geometry is not exact.  The points are released when
 * 1 <= fixed_point <= n - 2, n the number of points of view 0; then every view must hold the same n object points (else
 * FID_CALIB_E_RO_VIEWS), n <= FID_CALIB_RO_MAX_POINTS (else FID_CALIB_E_POINTS) and n_views <= FID_CALIB_RO_MAX_VIEWS (else
 * FID_CALIB_E_INPUT) and fewer free parameters than residuals (else FID_CALIB_E_RO_RESIDUALS); the 3 coordinates of point 0 and of point fixed_point and z of point n - 1 stay as given, the other
 * 3n - 7 are estimated with the camera.  Outputs besides fid_calibrate_camera's (host, optional): new_obj_points [n][3] (cv2's
 * newObjPoints) and std_obj_points [n][3] (stdDeviationsObjPoints; exactly 0 for the fixed coordinates); *released (optional)
 * = 1.  With fixed_point out of that range the call is fid_calibrate_camera (the same kernels and bits), *released = 0 and the
 * object outputs are left untouched.  Device memory of a released call: about 8 (9 + 3n)^2 bytes for the reduced system,
 * 48 (9 + 3n) min(n_views, 256) for its chunk of views and 1.6 kB per view plus 36 bytes per image point (at the caps, 1 024 points
 * x 4 096 views: 77 + 38 + 6.6 + 151 MB, about 273 MB). */
#define FID_CALIB_RO_MAX_POINTS 1024 /* per view, when releasing */
#define FID_CALIB_RO_MAX_VIEWS 4096  /* when releasing */
int fid_calibrate_camera_ro(int device, int n_views, const int32_t* offsets, const float* obj, const float* img, int width, int height, const fid_camera* guess,
                            int32_t flags, const fid_calib_criteria* criteria, fid_calib_result* result, double* rvecs, double* tvecs, double* std_extrinsics,
                            double* per_view_errors, fid_calib_stats* stats /* optional */, int fixed_point, float* new_obj_points, double* std_obj_points,
                            int* released);

/* ------------------------------------------------------------------------------------------------
 * Map bundle adjustment (after the calibration types it shares).
 * ---------------------------------------------------------------------------------------------- */
/* Bundle adjustment of a map instance from recorded marker corners (NEW -- DESIGN.md f16; the reference only folds per-marker
 * poses, map.cpp:152-320, and fid_map_refine works from relative poses without pixels; parity stated here and pinned against
 * scipy.optimize.least_squares on the same residuals, tests/test_hostsim_map_ba.py).
 *   input     a recorded sequence in fid_detect_pose_batch's dense layout: counts[n_frames], ids[n_frames][max_markers],
 *             corners[n_frames][max_markers][4][2] (float32); the camera (K, plumb_bob D); fiducial_len and the node's overrides
 *             as fid_pose takes them
 *   unknowns  every used frame's camera-from-map pose (R_f, t_f) (cv2's rvec / tvec convention) and every free entry's pose
 *             T_mapFid = (R_m, t_m).  Entries with variance 0 stay fixed (the origin of autoInit / add_fiducial); none gives
 *             FID_ERR_INVALID_ARG
 *   residual  per observation of marker m in frame f, 8 values pi(K, D, R_f (R_m o_k + t_m) + t_f) - c_fk, k = 0..3: pi =
 *             cv::projectPoints, o_k = getSingleMarkerObjectPoints at the marker's length (override or fiducial_len);
 *             rms = sqrt(sum |e|^2 / corners)
 *   counts    ids not in the map are ignored; an id seen twice in a frame drops every observation of it in that frame; frames
 *             without a mapped marker are unused; only markers and frames connected through co-visibility to a fixed entry
 *             take part, the others are left untouched and counted
 *   init      per frame solvePnP(ITERATIVE) of its mapped markers as one board whose object points are the map-frame corners
 *             narrowed to float32 (cv2.aruco.Board + matchImagePoints + cv2.solvePnP on that board), unless one marker's fid_pose
 *             composed with its map pose reprojects the frame's corners better (candidates with a corner behind the camera
 *             never count).  A fold's map is nearly but not
 *             exactly planar, where solvePnP's non-planar DLT can put the camera metres off; the single-marker candidates keep
 *             the start in the right basin.  A frame without any candidate is dropped (status 3)
 *   solver    Levenberg-Marquardt with fid_calibrate_camera's CvLevMarq schedule, diagonals damped by 1 + lambda, the update
 *             R <- R Exp(dtheta), t <- t + dt; every step eliminates the frames (Schur complement, dense over the free markers)
 *             and factors the reduced system on the device.  |p| of the relative-step test = sqrt(sum angle(R)^2 + |t|^2)
 * Output: the free entries' poses are written back in place (variances, observation counts and links are left alone; fixed
 * and unreached entries stay byte-identical; read_only_map is not consulted).  Optional host outputs: frame_rvecs / frame_tvecs
 * [n_frames][3] (0 for unused frames), frame_status [n_frames] (FID_BA_FRAME_*), std_entries [entries][6] in fid_map_entries
 * order: the standard deviations of (dtheta, dt) at the optimum, sqrt(sigma^2 diag(S^-1)) with sigma^2 = sum |e|^2 /
 * (2 corners - free parameters), 0 for fixed and unreached entries.  Device reruns are bit-identical (fixed summation orders, no
 * atomics).  stats->converged = 0 when the run stopped at max_iter rather than on the relative-step test (the poses are still
 * written back; the cost never rose).  Caps: FID_BA_MAX_FREE free markers, FID_BA_MAX_FRAMES frames, FID_BA_MAX_OBS
 * observations (FID_ERR_CAPACITY above, nothing written).  FID_ERR_INVALID_ARG for non-finite corners, a bad camera, bad sizes,
 * no fixed entry or a non-positive pivot (a pose the observations do not determine; nothing is written back then).  Waits for
 * pending asynchronous updates first.  Device memory: about 1.3 kB per observation (including the initial poses' staging),
 * 0.7 kB per frame, 8 bytes per pair of free markers seen together in a frame (the co-visibility lists: k markers per frame
 * give k (k - 1) / 2 pairs) and 8 mp (mp + min(6M, 768)) bytes for the reduced system, mp = 6M rounded up to 32 (at the caps,
 * 1 024 free markers: 302 + 38 MB, plus 5.5 GB for 2^22 observations). */
#define FID_BA_MAX_FREE 1024
#define FID_BA_MAX_FRAMES 65536
#define FID_BA_MAX_OBS (1 << 22)
#define FID_BA_FRAME_NONE 0      /* no mapped marker */
#define FID_BA_FRAME_USED 1
#define FID_BA_FRAME_UNREACHED 2 /* not connected to a fixed entry */
#define FID_BA_FRAME_INIT 3      /* dropped by the initial pose (solvePnP would raise) */
typedef struct fid_ba_params {
    /* type bit 1 = COUNT (max_iter, clamped to 1..1000; else 100), bit 2 = EPS (epsilon on the relative step; else 1e-12) */
    fid_calib_criteria criteria;
} fid_ba_params;
typedef struct fid_ba_stats {
    double initial_rms, final_rms; /* px, at the initial poses and at the optimum */
    double device_ms;              /* CUDA events around the device work (initial poses + solve) */
    int32_t iterations, n_steps;   /* CvLevMarq iterations and trial steps */
    int32_t frames_used, markers_used /* free markers solved */, observations_used;
    int32_t dropped_unmapped, dropped_duplicate; /* detections */
    int32_t frames_unreached, markers_unreached /* free entries not taking part */, frames_init_failed;
    int32_t kernel_launches;
    int32_t converged;             /* 1: the relative-step test ended the run; 0: it stopped at max_iter (poses still written back) */
} fid_ba_stats;
int fid_map_ba_default_params(fid_ba_params* p);
int fid_map_bundle_adjust(fid_map* m, int instance, int n_frames, const int32_t* counts, const int32_t* ids, const float* corners, int max_markers,
                          const fid_camera* cam, double fiducial_len, int n_override, const int32_t* override_ids, const double* override_lens,
                          const fid_ba_params* params /* NULL = defaults */, fid_ba_stats* stats /* optional */, double* frame_rvecs, double* frame_tvecs,
                          int32_t* frame_status, double* std_entries);

/* Localization against the map: one camera pose per frame from every visible mapped marker's corners together, with its
 * covariance (NEW -- DESIGN.md f17; the reference's updatePose, map.cpp:247-391, averages one pose per marker with heuristic
 * variances, and the `multi_error_theshold` it reads at :127-129 for a multi-fiducial pose is never used; stated here and pinned
 * against cv2, tests/test_hostsim_map_localize.py).  Per frame f of the dense fid_detect_pose_batch layout (counts, ids, corners):
 *   match     a detection counts when its id is in the map instance, appears once in the frame, and (max_entry_variance >= 0)
 *             the entry's variance is <= max_entry_variance; detection order is kept
 *   board     each counted marker's getSingleMarkerObjectPoints at its length (override or fiducial_len) through its entry's
 *             pose, narrowed to float32: the cv2.aruco.Board of the map's markers
 *   start     fid_map_bundle_adjust's initial pose: the board's solvePnP(ITERATIVE), unless one marker's own fid_pose composed
 *             with its map pose reprojects all the frame's corners better (candidates with a corner behind the camera never
 *             count).  start = 0 (board) or 1 + k (the k-th counted marker); none: status FID_LOC_NO_START
 *   LM        cv2.solvePnP(obj, img, K, D, rvec0, tvec0, useExtrinsicGuess=True, SOLVEPNP_ITERATIVE) from that start: rvec, tvec
 *             (camera-from-map), lm_iters; image_error = mean squared reprojection error with float32-rounded projections
 *   pose      t, q (x y z w): T_mapBase = T_mapCam T_camBase when T_camBase is given (have_base = 1; updatePose's composition,
 *             map.cpp:284), else T_mapCam
 *   cov       row-major 6x6 over (x, y, z, rotation about map X, Y, Z) of that pose (ROS PoseWithCovariance order) for the
 *             perturbation (Exp([dtheta]x) R, t + dt): sigma2 (J^T J)^-1, J the Jacobian of every corner residual at the final
 *             pose, sigma2 = sum |e|^2 / (2 n_points - 6); cov_ok = 0 and a zero covariance on a non-positive Cholesky pivot
 *   object_error  (image_error / mean |c0 - c2| px) (mean |marker centre in the camera frame| / fiducial_len) over the counted
 *             markers: aruco_detect.cpp:493-495's formula at the joint pose, the quantity multi_error_theshold is compared with
 * out[n_frames].  FID_ERR_INVALID_ARG for a bad camera, non-finite corners, counts[f] outside 0..max_markers, max_markers outside
 * 1..FID_MAX_MARKERS, non-positive lengths or a bad instance; FID_ERR_CAPACITY above FID_BA_MAX_FRAMES frames; nothing is
 * written then.  The map is not changed.  Runs on the map's stream after pending asynchronous updates; device reruns are
 * bit-identical (a warp per frame, fixed summation orders, no atomics). */
#define FID_LOC_POSE 1
#define FID_LOC_NONE 0      /* no usable mapped marker */
#define FID_LOC_NO_START (-1)
typedef struct fid_localization {
    int32_t status, n_markers, n_points, lm_iters, start, have_base, cov_ok;
    double rvec[3], tvec[3], t[3], q[4], image_error, object_error, sigma2, covariance[36];
} fid_localization;
int fid_map_localize(fid_map* m, int instance, int n_frames, const int32_t* counts, const int32_t* ids, const float* corners, int max_markers,
                     const fid_camera* cam, double fiducial_len, int n_override, const int32_t* override_ids, const double* override_lens,
                     double max_entry_variance, const fid_tf* T_camBase /* NULL: camera pose only */, fid_localization* out /* [n_frames] */);

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
