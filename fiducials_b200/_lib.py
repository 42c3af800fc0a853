"""ctypes binding of libfiducials_b200.so (include/fiducials_b200.h).

The library is built in-tree by ``__graft_entry__.build()`` / ``fiducials_b200/build.py``.  There is
no fallback: if the shared object is missing, or no CUDA device is usable, the calls raise.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libfiducials_b200.so")

FID_OK = 0
FID_MAX_MARKERS = 256


class FidError(RuntimeError):
    def __init__(self, status, what=""):
        self.status = status
        msg = "fiducials_b200 error %d" % status
        if _lib is not None:
            msg += ": " + _lib.fid_strerror(status).decode()
        super().__init__(msg + (" (%s)" % what if what else ""))


class fid_params(C.Structure):
    _fields_ = [
        ("dictionary", C.c_int32),
        ("adaptiveThreshConstant", C.c_double),
        ("adaptiveThreshWinSizeMax", C.c_int32),
        ("adaptiveThreshWinSizeMin", C.c_int32),
        ("adaptiveThreshWinSizeStep", C.c_int32),
        ("cornerRefinementMaxIterations", C.c_int32),
        ("cornerRefinementMinAccuracy", C.c_double),
        ("cornerRefinementWinSize", C.c_int32),
        ("cornerRefinementMethod", C.c_int32),
        ("errorCorrectionRate", C.c_double),
        ("minCornerDistanceRate", C.c_double),
        ("markerBorderBits", C.c_int32),
        ("maxErroneousBitsInBorderRate", C.c_double),
        ("minDistanceToBorder", C.c_int32),
        ("minMarkerDistanceRate", C.c_double),
        ("minMarkerPerimeterRate", C.c_double),
        ("maxMarkerPerimeterRate", C.c_double),
        ("minOtsuStdDev", C.c_double),
        ("perspectiveRemoveIgnoredMarginPerCell", C.c_double),
        ("perspectiveRemovePixelPerCell", C.c_int32),
        ("polygonalApproxAccuracyRate", C.c_double),
        ("relativeCornerRefinmentWinSize", C.c_double),
        ("minGroupDistance", C.c_double),
    ]


class fid_camera(C.Structure):
    _fields_ = [("K", C.c_double * 9), ("D", C.c_double * 5)]


class fid_transform(C.Structure):
    _fields_ = [
        ("fiducial_id", C.c_int32),
        ("reserved", C.c_int32),
        ("translation", C.c_double * 3),
        ("rotation", C.c_double * 4),
        ("image_error", C.c_double),
        ("object_error", C.c_double),
        ("fiducial_area", C.c_double),
        ("rvec", C.c_double * 3),
    ]


class fid_pose_hypotheses(C.Structure):
    """struct fid_pose_hypotheses: both planar (IPPE_SQUARE) pose solutions of a marker, solvePnPGeneric's order."""
    _fields_ = [
        ("fiducial_id", C.c_int32),
        ("n", C.c_int32),
        ("iterative_match", C.c_int32),
        ("reserved", C.c_int32),
        ("rvec", (C.c_double * 3) * 2),
        ("tvec", (C.c_double * 3) * 2),
        ("rms", C.c_double * 2),
    ]


class fid_board(C.Structure):
    """fid_board: the markers of one board, as fid_set_boards takes them."""
    _fields_ = [
        ("n_markers", C.c_int32),
        ("ids", C.c_void_p),
        ("obj_points", C.c_void_p),
    ]


class fid_board_pose(C.Structure):
    """fid_board_pose: one pose per board (Board::matchImagePoints + solvePnP(SOLVEPNP_ITERATIVE))."""
    _fields_ = [
        ("board", C.c_int32),
        ("status", C.c_int32),
        ("n_markers", C.c_int32),
        ("n_points", C.c_int32),
        ("rvec", C.c_double * 3),
        ("tvec", C.c_double * 3),
        ("rotation", C.c_double * 4),
        ("image_error", C.c_double),
    ]


class fid_charuco_board(C.Structure):
    """fid_charuco_board: one ChArUco board, as fid_set_charuco_boards takes it."""
    _fields_ = [
        ("squares_x", C.c_int32),
        ("squares_y", C.c_int32),
        ("square_length", C.c_float),
        ("marker_length", C.c_float),
        ("legacy_pattern", C.c_int32),
        ("ids", C.c_void_p),
        ("min_markers", C.c_int32),
        ("check_markers", C.c_int32),
    ]


class fid_charuco_result(C.Structure):
    """fid_charuco_result: the corners and pose of one (frame, ChArUco board)."""
    _fields_ = [
        ("board", C.c_int32),
        ("n_corners", C.c_int32),
        ("corner_offset", C.c_int32),
        ("status", C.c_int32),
        ("rvec", C.c_double * 3),
        ("tvec", C.c_double * 3),
        ("rotation", C.c_double * 4),
        ("image_error", C.c_double),
    ]


class fid_marker_refine_params(C.Structure):
    """fid_marker_refine_params: cv::aruco::RefineParameters of the recovery of missed board markers."""
    _fields_ = [
        ("enable", C.c_int32),
        ("min_rep_distance", C.c_float),
        ("error_correction_rate", C.c_float),
        ("check_all_orders", C.c_int32),
    ]


FID_MAX_REJECTED = 4096


class fid_diamond_params(C.Structure):
    """fid_diamond_params: the ChArUco diamond geometry and the CharucoParameters its detection uses."""
    _fields_ = [
        ("enable", C.c_int32),
        ("square_length", C.c_float),
        ("marker_length", C.c_float),
        ("min_markers", C.c_int32),
        ("check_markers", C.c_int32),
    ]


class fid_diamond(C.Structure):
    """fid_diamond: one ChArUco diamond (cv2's diamondIds and diamondCorners) and its pose."""
    _fields_ = [
        ("ids", C.c_int32 * 4),
        ("corners", C.c_float * 8),
        ("status", C.c_int32),
        ("pose", fid_transform),
    ]


FID_MAX_DIAMONDS = 64
FID_MAX_DICTIONARIES = 8


class fid_dictionary_spec(C.Structure):
    """fid_dictionary_spec: one entry of a multi-dictionary detector (fid_set_dictionaries)."""
    _fields_ = [("dictionary", C.c_int32), ("id_offset", C.c_int32), ("fiducial_len", C.c_double)]


class fid_aruco3_params(C.Structure):
    """fid_aruco3_params: useAruco3Detection (fid_set_aruco3)."""
    _fields_ = [("enable", C.c_int32), ("minSideLengthCanonicalImg", C.c_int32), ("minMarkerLengthRatioOriginalImg", C.c_double)]


class fid_calib_criteria(C.Structure):
    _fields_ = [("type", C.c_int32), ("max_iter", C.c_int32), ("epsilon", C.c_double)]


class fid_calib_result(C.Structure):
    _fields_ = [("rms", C.c_double), ("camera", fid_camera), ("std_intrinsics", C.c_double * 9), ("iterations", C.c_int32), ("status", C.c_int32)]


FID_CALIB_MAX_STEPS = 2048


class fid_calib_stats(C.Structure):
    _fields_ = [("n_steps", C.c_int32), ("n_evaluations", C.c_int32), ("kernel_launches", C.c_int32), ("reserved", C.c_int32), ("device_ms", C.c_double),
                ("steps", C.c_uint8 * FID_CALIB_MAX_STEPS)]


class fid_map_params(C.Structure):
    _fields_ = [
        ("weighting_scale", C.c_double),
        ("use_fiducial_area_as_weight", C.c_int32),
        ("read_only_map", C.c_int32),
        ("systematic_error", C.c_double),
        ("max_fiducials", C.c_int32),
        ("n_instances", C.c_int32),
    ]


class fid_map_file_entry(C.Structure):
    _fields_ = [("fiducial_id", C.c_int32), ("num_obs", C.c_int32)] + [(k, C.c_double) for k in ("x", "y", "z", "roll_deg", "pitch_deg", "yaw_deg", "variance")]


class fid_tf(C.Structure):
    _fields_ = [("t", C.c_double * 3), ("q", C.c_double * 4)]


class fid_robot_pose(C.Structure):
    _fields_ = [("valid", C.c_int32), ("n_estimates", C.c_int32), ("t", C.c_double * 3), ("q", C.c_double * 4), ("variance", C.c_double)]


class fid_ba_params(C.Structure):
    _fields_ = [("criteria", fid_calib_criteria)]


class fid_ba_stats(C.Structure):
    _fields_ = [("initial_rms", C.c_double), ("final_rms", C.c_double), ("device_ms", C.c_double)] + [(k, C.c_int32) for k in (
        "iterations", "n_steps", "frames_used", "markers_used", "observations_used", "dropped_unmapped", "dropped_duplicate", "frames_unreached", "markers_unreached",
        "frames_init_failed", "kernel_launches", "converged")]


class fid_localization(C.Structure):
    _fields_ = [(k, C.c_int32) for k in ("status", "n_markers", "n_points", "lm_iters", "start", "have_base", "cov_ok")] + [
        ("rvec", C.c_double * 3), ("tvec", C.c_double * 3), ("t", C.c_double * 3), ("q", C.c_double * 4), ("image_error", C.c_double), ("object_error", C.c_double),
        ("sigma2", C.c_double), ("covariance", C.c_double * 36)]


class fid_map_entry(C.Structure):
    _fields_ = [("fiducial_id", C.c_int32), ("num_obs", C.c_int32)] + [(k, C.c_double) for k in ("x", "y", "z", "rx", "ry", "rz", "variance")]


class fid_refine_params(C.Structure):
    _fields_ = [("max_iterations", C.c_int32), ("pcg_iterations", C.c_int32), ("pcg_tolerance", C.c_double), ("damping", C.c_double), ("translation_weight", C.c_double)]


class fid_refine_stats(C.Structure):
    _fields_ = [("initial_cost", C.c_double), ("final_cost", C.c_double), ("solve_ms", C.c_double), ("iterations", C.c_int32), ("n_edges", C.c_int32), ("n_free", C.c_int32), ("kernel_launches", C.c_int32)]


class fid_map_record(C.Structure):
    _fields_ = [("fiducial_id", C.c_int32), ("num_obs", C.c_int32), ("t", C.c_double * 3), ("q", C.c_double * 4), ("variance", C.c_double)]


# every symbol include/fiducials_b200.h declares (tests/test_abi.py checks the list against the header)
EXPORTS = [
    "fid_strerror", "fid_version", "fid_default_params", "fid_create", "fid_destroy", "fid_set_params", "fid_detect", "fid_pose",
    "fid_detect_pose_batch", "fid_submit_batch", "fid_collect_batch", "fid_set_pose_hypotheses", "fid_pose_hypotheses", "fid_last_pose_hypotheses", "fid_set_boards", "fid_estimate_board_poses", "fid_last_board_poses", "fid_set_charuco_boards", "fid_detect_charuco", "fid_last_charuco", "fid_set_marker_refinement", "fid_refine_detected_markers", "fid_set_batch_marker_refinement", "fid_last_marker_refinement", "fid_set_diamonds", "fid_detect_diamonds", "fid_last_diamonds", "fid_set_dictionaries", "fid_set_family_boards", "fid_set_family_charuco_boards", "fid_set_family_diamonds", "fid_detect_multi_dict", "fid_last_dict_indices", "fid_set_aruco3", "fid_debug_aruco3_planes", "fid_detect_with_confidence", "fid_set_marker_confidence", "fid_last_marker_confidence", "fid_set_detect_inverted_marker", "fid_hint_next", "fid_set_input_encoding", "fid_timer_start", "fid_timer_stop", "fid_host_alloc", "fid_host_free", "fid_device_alloc", "fid_device_free", "fid_memcpy_h2d", "fid_debug_threshold", "fid_debug_time_threshold",
    "fid_debug_candidates", "fid_debug_rejected", "fid_last_stage_ms", "fid_last_counters", "fid_map_default_params", "fid_map_create", "fid_map_destroy", "fid_map_clear",
    "fid_map_load", "fid_map_links", "fid_map_add_links", "fid_map_update", "fid_map_update_sequence", "fid_map_update_frames", "fid_map_update_frames_async", "fid_map_sync", "fid_map_entries", "fid_map_export", "fid_map_merge", "fid_map_export_device",
    "fid_map_merge_device", "fid_map_merge_device_async", "fid_map_export_async", "fid_map_stream", "fid_map_merged_entries", "fid_map_adopt_merged", "fid_map_add_fiducial", "fid_map_refine_default_params", "fid_map_refine",
    "fid_jpeg_create", "fid_jpeg_destroy", "fid_jpeg_decode_batch", "fid_jpeg_sync", "fid_jpeg_stream", "fid_jpeg_last_stats", "fid_calibrate_camera",
    "fid_calibrate_camera_ro", "fid_map_ba_default_params", "fid_map_bundle_adjust", "fid_map_localize",
]

_lib = None


def load():
    """Load libfiducials_b200.so or raise.  (Built by __graft_entry__.build().)"""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise FileNotFoundError("%s not found -- run `python -c 'import __graft_entry__ as g; g.build()'` (no CPU fallback exists)" % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    lib.fid_strerror.restype = C.c_char_p
    lib.fid_strerror.argtypes = [C.c_int]
    lib.fid_version.restype = C.c_char_p
    vp, i32, sz = C.c_void_p, C.c_int, C.c_size_t
    lib.fid_default_params.argtypes = [C.POINTER(fid_params)]
    lib.fid_create.argtypes = [C.POINTER(fid_params), i32, i32, i32, i32, C.POINTER(vp)]
    lib.fid_destroy.argtypes = [vp]
    lib.fid_set_params.argtypes = [vp, C.POINTER(fid_params)]
    lib.fid_detect.argtypes = [vp, vp, i32, i32, sz, i32, C.POINTER(i32), vp, vp]
    lib.fid_pose.argtypes = [vp, i32, vp, vp, C.POINTER(fid_camera), C.c_double, i32, vp, vp, vp]
    lib.fid_detect_pose_batch.argtypes = [vp, i32, vp, i32, i32, i32, sz, sz, C.POINTER(fid_camera), C.c_double, i32, vp, vp, i32, vp, vp, vp, vp]
    lib.fid_submit_batch.argtypes = [vp, i32, vp, i32, i32, i32, sz, sz, C.POINTER(fid_camera), C.c_double, i32, vp, vp]
    lib.fid_collect_batch.argtypes = [vp, i32, vp, vp, vp, vp]
    lib.fid_set_pose_hypotheses.argtypes = [vp, i32]
    lib.fid_pose_hypotheses.argtypes = [vp, i32, vp, vp, C.POINTER(fid_camera), C.c_double, i32, vp, vp, vp]
    lib.fid_last_pose_hypotheses.argtypes = [vp, i32, C.POINTER(i32), vp]
    lib.fid_set_boards.argtypes = [vp, i32, vp]
    lib.fid_estimate_board_poses.argtypes = [vp, i32, vp, vp, C.POINTER(fid_camera), vp]
    lib.fid_last_board_poses.argtypes = [vp, i32, C.POINTER(i32), C.POINTER(i32), vp]
    lib.fid_set_charuco_boards.argtypes = [vp, i32, vp]
    lib.fid_detect_charuco.argtypes = [vp, vp, i32, i32, sz, i32, vp, vp, C.POINTER(fid_camera), vp, vp, vp]
    lib.fid_last_charuco.argtypes = [vp, i32, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32), vp, vp, vp]
    lib.fid_set_marker_refinement.argtypes = [vp, C.POINTER(fid_marker_refine_params)]
    lib.fid_refine_detected_markers.argtypes = [vp, vp, i32, i32, sz, i32, vp, vp, i32, i32, vp, C.POINTER(fid_camera), C.POINTER(i32), vp, vp]
    lib.fid_set_batch_marker_refinement.argtypes = [vp, i32]
    lib.fid_last_marker_refinement.argtypes = [vp, i32, i32, C.POINTER(i32), vp, vp, vp, vp, vp]
    lib.fid_set_diamonds.argtypes = [vp, C.POINTER(fid_diamond_params)]
    lib.fid_detect_diamonds.argtypes = [vp, vp, i32, i32, sz, i32, vp, vp, C.POINTER(fid_camera), C.POINTER(i32), vp]
    lib.fid_last_diamonds.argtypes = [vp, i32, C.POINTER(i32), vp, vp]
    lib.fid_set_dictionaries.argtypes = [vp, i32, vp]
    lib.fid_set_family_boards.argtypes = [vp, i32, vp, vp]
    lib.fid_set_family_charuco_boards.argtypes = [vp, i32, vp, vp]
    lib.fid_set_family_diamonds.argtypes = [vp, C.POINTER(fid_diamond_params), C.c_int32]
    lib.fid_detect_multi_dict.argtypes = [vp, vp, i32, i32, sz, i32, C.POINTER(i32), vp, vp, vp]
    lib.fid_last_dict_indices.argtypes = [vp, i32, C.POINTER(i32), vp]
    lib.fid_set_aruco3.argtypes = [vp, C.POINTER(fid_aruco3_params)]
    lib.fid_debug_aruco3_planes.argtypes = [vp, vp, i32, i32, sz, vp, vp, vp, sz]
    lib.fid_detect_with_confidence.argtypes = [vp, vp, i32, i32, sz, i32, C.POINTER(i32), vp, vp, vp]
    lib.fid_set_marker_confidence.argtypes = [vp, i32]
    lib.fid_last_marker_confidence.argtypes = [vp, i32, C.POINTER(i32), vp]
    lib.fid_set_detect_inverted_marker.argtypes = [vp, i32]
    lib.fid_hint_next.argtypes = [vp, vp]
    lib.fid_set_input_encoding.argtypes = [vp, i32]
    lib.fid_debug_time_threshold.argtypes = [vp, i32, vp, i32, i32, sz, sz, i32, C.POINTER(C.c_float)]
    lib.fid_timer_start.argtypes = [vp]
    lib.fid_timer_stop.argtypes = [vp, C.POINTER(C.c_float)]
    lib.fid_host_alloc.argtypes = [sz, C.POINTER(vp)]
    lib.fid_host_free.argtypes = [vp]
    lib.fid_device_alloc.argtypes = [vp, sz, C.POINTER(vp)]
    lib.fid_device_free.argtypes = [vp, vp]
    lib.fid_memcpy_h2d.argtypes = [vp, vp, vp, sz]
    lib.fid_debug_threshold.argtypes = [vp, vp, i32, i32, sz, vp, vp, C.POINTER(i32)]
    lib.fid_debug_candidates.argtypes = [vp, i32, C.POINTER(i32), vp, vp, vp]
    lib.fid_debug_rejected.argtypes = [vp, i32, C.POINTER(i32), vp]
    lib.fid_last_stage_ms.argtypes = [vp, vp, i32, C.POINTER(i32)]
    lib.fid_last_counters.argtypes = [vp, vp, i32, C.POINTER(i32)]
    lib.fid_map_default_params.argtypes = [C.POINTER(fid_map_params)]
    lib.fid_map_create.argtypes = [C.POINTER(fid_map_params), i32, C.POINTER(vp)]
    lib.fid_map_destroy.argtypes = [vp]
    lib.fid_map_clear.argtypes = [vp, i32]
    lib.fid_map_load.argtypes = [vp, i32, i32, vp]
    lib.fid_map_links.argtypes = [vp, i32, i32, C.POINTER(C.c_int), vp]
    lib.fid_map_add_links.argtypes = [vp, i32, i32, vp]
    lib.fid_map_update.argtypes = [vp, i32, i32, vp, C.POINTER(fid_tf), C.POINTER(fid_tf), C.POINTER(fid_robot_pose)]
    lib.fid_map_update_sequence.argtypes = [vp, i32, vp, vp, C.POINTER(fid_tf), C.POINTER(fid_tf), vp]
    lib.fid_map_update_frames.argtypes = [vp, i32, i32, vp, vp, i32, C.POINTER(fid_tf), C.POINTER(fid_tf), C.POINTER(fid_robot_pose)]
    lib.fid_map_update_frames_async.argtypes = [vp, i32, i32, vp, vp, i32, C.POINTER(fid_tf), C.POINTER(fid_tf)]
    lib.fid_map_sync.argtypes = [vp]
    lib.fid_map_entries.argtypes = [vp, i32, i32, C.POINTER(i32), vp]
    lib.fid_map_export.argtypes = [vp, i32, vp]
    lib.fid_map_merge.argtypes = [vp, i32, vp]
    lib.fid_map_export_device.argtypes = [vp, i32, C.POINTER(vp), C.POINTER(sz)]
    lib.fid_map_merge_device.argtypes = [vp, i32, vp]
    lib.fid_map_merge_device_async.argtypes = [vp, i32, vp]
    lib.fid_map_export_async.argtypes = [vp, i32, vp]
    lib.fid_map_stream.argtypes = [vp, C.POINTER(vp)]
    lib.fid_map_merged_entries.argtypes = [vp, i32, C.POINTER(C.c_int), vp]
    lib.fid_map_adopt_merged.argtypes = [vp, i32]
    lib.fid_map_add_fiducial.argtypes = [vp, i32, i32, C.POINTER(fid_tf)]
    lib.fid_map_refine_default_params.argtypes = [C.POINTER(fid_refine_params)]
    lib.fid_map_refine.argtypes = [vp, i32, i32, vp, vp, C.POINTER(fid_refine_params), C.POINTER(fid_refine_stats)]
    lib.fid_jpeg_create.argtypes = [i32, i32, i32, i32, i32, C.POINTER(vp)]
    lib.fid_jpeg_destroy.argtypes = [vp]
    lib.fid_jpeg_decode_batch.argtypes = [vp, i32, vp, vp, i32, i32, vp, sz, sz, vp]
    lib.fid_jpeg_sync.argtypes = [vp]
    lib.fid_jpeg_stream.argtypes = [vp, C.POINTER(vp)]
    lib.fid_jpeg_last_stats.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double)]
    lib.fid_calibrate_camera.argtypes = [i32, i32, vp, vp, vp, i32, i32, C.POINTER(fid_camera), i32, C.POINTER(fid_calib_criteria), C.POINTER(fid_calib_result), vp, vp,
                                         vp, vp, C.POINTER(fid_calib_stats)]
    lib.fid_calibrate_camera_ro.argtypes = lib.fid_calibrate_camera.argtypes + [i32, vp, vp, C.POINTER(C.c_int)]
    lib.fid_map_ba_default_params.argtypes = [C.POINTER(fid_ba_params)]
    lib.fid_map_bundle_adjust.argtypes = [vp, i32, i32, vp, vp, vp, i32, C.POINTER(fid_camera), C.c_double, i32, vp, vp, C.POINTER(fid_ba_params), C.POINTER(fid_ba_stats),
                                          vp, vp, vp, vp]
    lib.fid_map_localize.argtypes = [vp, i32, i32, vp, vp, vp, i32, C.POINTER(fid_camera), C.c_double, i32, vp, vp, C.c_double, C.POINTER(fid_tf),
                                     C.POINTER(fid_localization)]
    for name in EXPORTS:
        getattr(lib, name)  # AttributeError if the build lost a symbol
    _lib = lib
    return lib


def check(status, what=""):
    if status != FID_OK:
        raise FidError(status, what)
