"""Host-side mirror of the reference's two nodes over the C-ABI (include/fiducials_b200.h).

``FiducialsNode`` follows aruco_detect/src/aruco_detect.cpp (FiducialsNode: camInfoCallback :307-330,
imageCallback :332-395, poseEstimateCallback :397-538, ignore list :540-571, length overrides
:627-660); ``FiducialSlam`` follows fiducial_slam/src/fiducial_slam.cpp (transformCallback :79-105)
and Map (map.cpp).  Same names, same argument meaning, same error behaviour (a frame that cannot be
processed is dropped and an empty/None result returned, never an exception from the callbacks);
the arithmetic happens on the GPU inside libfiducials_b200.so.  This python layer exists for the
parity tests and bench.py; the C++ twin for a real ROS node is fiducials_b200/csrc/node_glue.hpp.
"""
from __future__ import annotations

import ctypes as C
import math
import re
from typing import Dict, Iterable, List, Optional, Sequence

import numpy as np

from . import _lib
from .msgs import (Detection2D, Detection2DArray, ObjectHypothesisWithPose, Fiducial, FiducialArray, FiducialMapEntry, FiducialMapEntryArray, FiducialTransform, FiducialTransformArray, Header, Transform)

MAXM = _lib.FID_MAX_MARKERS


def default_params(**overrides) -> "_lib.fid_params":
    lib = _lib.load()
    p = _lib.fid_params()
    _lib.check(lib.fid_default_params(C.byref(p)))
    for k, v in overrides.items():
        if not hasattr(p, k):
            raise AttributeError("unknown detector parameter %r" % k)
        setattr(p, k, v)
    return p


def _camera(K, D) -> "_lib.fid_camera":
    cam = _lib.fid_camera()
    K = np.asarray(K, np.float64).reshape(9)
    D = np.asarray(D, np.float64).reshape(-1)
    for i in range(9):
        cam.K[i] = float(K[i])
    for i in range(5):
        cam.D[i] = float(D[i]) if i < len(D) else 0.0  # first five coefficients (:317-323)
    return cam


class Detector:
    """Thin RAII wrapper of fid_detector*."""

    def __init__(self, params=None, device=0, max_width=1920, max_height=1080, max_batch=1):
        self.lib = _lib.load()
        self.params = params if params is not None else default_params()
        self.bpp = 3
        self.h = C.c_void_p()
        _lib.check(self.lib.fid_create(C.byref(self.params), device, max_width, max_height, max_batch, C.byref(self.h)), "fid_create")
        self.max_batch = max_batch
        self.max_width, self.max_height = max_width, max_height

    def close(self):
        if getattr(self, "h", None) is not None and self.h.value:
            self.lib.fid_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_params(self, params):
        _lib.check(self.lib.fid_set_params(self.h, C.byref(params)))
        self.params = params

    ENCODINGS = {"bgr8": 0, "rgb8": 1, "mono8": 2}

    def set_input_encoding(self, encoding: str):
        """fid_set_input_encoding: the camera's own sensor_msgs/Image encoding ("bgr8", "rgb8", "mono8"; frames are then
        [n,H,W,3] or [n,H,W]) instead of the BGR8 copy cv_bridge makes for the reference (aruco_detect.cpp:348)."""
        _lib.check(self.lib.fid_set_input_encoding(self.h, self.ENCODINGS[encoding]), "fid_set_input_encoding")
        self.bpp = 1 if encoding == "mono8" else 3

    def detect(self, bgr: np.ndarray):
        """fid_detect: (ids int32[n], corners float32[n,4,2])."""
        bgr = np.ascontiguousarray(bgr, np.uint8)
        H, W = bgr.shape[:2]
        ids = np.zeros(MAXM, np.int32)
        corners = np.zeros((MAXM, 8), np.float32)
        n = C.c_int(0)
        _lib.check(self.lib.fid_detect(self.h, bgr.ctypes.data_as(C.c_void_p), W, H, W * self.bpp, MAXM, C.byref(n), ids.ctypes.data_as(C.c_void_p),
                                       corners.ctypes.data_as(C.c_void_p)), "fid_detect")
        return ids[: n.value].copy(), corners[: n.value].reshape(-1, 4, 2).copy()

    def pose(self, ids, corners, K, D, fiducial_len, overrides: Optional[Dict[int, float]] = None):
        ids = np.ascontiguousarray(ids, np.int32)
        corners = np.ascontiguousarray(corners, np.float32).reshape(-1, 8)
        n = len(ids)
        out = (_lib.fid_transform * max(n, 1))()
        cam = _camera(K, D)
        oi, ol, no = _overrides(overrides)
        _lib.check(self.lib.fid_pose(self.h, n, ids.ctypes.data_as(C.c_void_p), corners.ctypes.data_as(C.c_void_p), C.byref(cam), float(fiducial_len), no,
                                     oi.ctypes.data_as(C.c_void_p), ol.ctypes.data_as(C.c_void_p), C.cast(out, C.c_void_p)), "fid_pose")
        return [out[i] for i in range(n)]

    def detect_pose_batch(self, frames, K=None, D=None, fiducial_len=0.14, overrides=None, on_device=False, n_frames=None, width=None, height=None):
        """frames: uint8 array [n,H,W,3] (host) or an integer device address when on_device.
        Returns counts[n], ids[n,MAXM], corners[n,MAXM,4,2], transforms (ctypes array n*MAXM or None)."""
        if on_device:
            n, H, W = int(n_frames), int(height), int(width)
            ptr = C.c_void_p(int(frames))
        else:
            frames = np.ascontiguousarray(frames, np.uint8)
            n, H, W = frames.shape[:3]
            ptr = frames.ctypes.data_as(C.c_void_p)
        cam = _camera(K, D) if K is not None else None
        key = (n, cam is not None)
        if getattr(self, "_out_key", None) != key:  # output buffers are reused between calls of the same shape
            self._out = (np.zeros(n, np.int32), np.zeros((n, MAXM), np.int32), np.zeros((n, MAXM, 8), np.float32),
                         (_lib.fid_transform * (n * MAXM))() if cam is not None else None)
            self._out_key = key
        counts, ids, corners, tfs = self._out
        oi, ol, no = _overrides(overrides)
        st = self.lib.fid_detect_pose_batch(self.h, n, ptr, 1 if on_device else 0, W, H, W * self.bpp, W * self.bpp * H, C.byref(cam) if cam is not None else None, float(fiducial_len), no,
                                            oi.ctypes.data_as(C.c_void_p), ol.ctypes.data_as(C.c_void_p), MAXM, counts.ctypes.data_as(C.c_void_p),
                                            ids.ctypes.data_as(C.c_void_p), corners.ctypes.data_as(C.c_void_p), C.cast(tfs, C.c_void_p) if tfs is not None else None)
        _lib.check(st, "fid_detect_pose_batch")
        return counts, ids, corners.reshape(n, MAXM, 4, 2), tfs

    def submit_batch(self, frames, K=None, D=None, fiducial_len=0.14, overrides=None, on_device=False, n_frames=None, width=None, height=None):
        """fid_submit_batch: queue a batch and return at once (see detect_pose_batch for the arguments).  Host frames must
        stay alive and unchanged until the matching collect_batch."""
        if on_device:
            n, H, W = int(n_frames), int(height), int(width)
            ptr = C.c_void_p(int(frames))
        else:
            assert frames.dtype == np.uint8 and frames.flags["C_CONTIGUOUS"]
            n, H, W = frames.shape[:3]
            ptr = frames.ctypes.data_as(C.c_void_p)
        cam = _camera(K, D) if K is not None else None
        oi, ol, no = _overrides(overrides)
        _lib.check(self.lib.fid_submit_batch(self.h, n, ptr, 1 if on_device else 0, W, H, W * self.bpp, W * self.bpp * H, C.byref(cam) if cam is not None else None, float(fiducial_len), no,
                                             oi.ctypes.data_as(C.c_void_p), ol.ctypes.data_as(C.c_void_p)), "fid_submit_batch")
        if not hasattr(self, "_pending"):
            self._pending = []
        self._pending.append((n, cam is not None, frames))

    def collect_batch(self, out=None):
        """fid_collect_batch: results of the oldest submitted batch, as detect_pose_batch returns them.  `out` = a tuple
        returned by an earlier call of the same shape, to reuse its buffers."""
        n, with_pose, _keep = self._pending.pop(0)
        if out is None:
            out = (np.zeros(n, np.int32), np.zeros((n, MAXM), np.int32), np.zeros((n, MAXM, 4, 2), np.float32), (_lib.fid_transform * (n * MAXM))() if with_pose else None)
        counts, ids, corners, tfs = out
        _lib.check(self.lib.fid_collect_batch(self.h, MAXM, counts.ctypes.data_as(C.c_void_p), ids.ctypes.data_as(C.c_void_p), corners.ctypes.data_as(C.c_void_p),
                                              C.cast(tfs, C.c_void_p) if tfs is not None else None), "fid_collect_batch")
        return counts, ids, corners, tfs

    def set_dictionaries(self, specs):
        """fid_set_dictionaries: specs = [(dictionary, id_offset, fiducial_len), ...] (a bare int is (dictionary, 0, 0.0)); entry 0's
        dictionary becomes params.dictionary.  Batches then detect with every dictionary (detectMarkersMultiDict)."""
        specs = [(s, 0, 0.0) if isinstance(s, (int, np.integer)) else tuple(s) for s in specs]
        arr = (_lib.fid_dictionary_spec * max(len(specs), 1))()
        for i, (d, off, ln) in enumerate(specs):
            arr[i] = _lib.fid_dictionary_spec(int(d), int(off), float(ln))
        _lib.check(self.lib.fid_set_dictionaries(self.h, len(specs), C.cast(arr, C.c_void_p)), "fid_set_dictionaries")
        self.params.dictionary = int(specs[0][0])

    def detect_multi_dict(self, bgr: np.ndarray):
        """fid_detect_multi_dict: (ids int32[n], corners float32[n,4,2], dict_indices int32[n])."""
        bgr = np.ascontiguousarray(bgr, np.uint8)
        H, W = bgr.shape[:2]
        ids = np.zeros(MAXM, np.int32)
        corners = np.zeros((MAXM, 8), np.float32)
        di = np.zeros(MAXM, np.int32)
        n = C.c_int(0)
        _lib.check(self.lib.fid_detect_multi_dict(self.h, bgr.ctypes.data_as(C.c_void_p), W, H, W * self.bpp, MAXM, C.byref(n), ids.ctypes.data_as(C.c_void_p),
                                                  corners.ctypes.data_as(C.c_void_p), di.ctypes.data_as(C.c_void_p)), "fid_detect_multi_dict")
        return ids[: n.value].copy(), corners[: n.value].reshape(-1, 4, 2).copy(), di[: n.value].copy()

    def last_dict_indices(self, max_markers=MAXM):
        """fid_last_dict_indices: int32 [n_frames, max_markers], laid out like the batch's ids."""
        nf = C.c_int(0)
        _lib.check(self.lib.fid_last_dict_indices(self.h, max_markers, C.byref(nf), None), "fid_last_dict_indices")
        out = np.zeros((nf.value, max_markers), np.int32)
        _lib.check(self.lib.fid_last_dict_indices(self.h, max_markers, C.byref(nf), out.ctypes.data_as(C.c_void_p)), "fid_last_dict_indices")
        return out

    def detect_with_confidence(self, bgr: np.ndarray):
        """fid_detect_with_confidence (detectMarkersWithConfidence): (ids int32[n], corners float32[n,4,2], confidence float32[n])."""
        bgr = np.ascontiguousarray(bgr, np.uint8)
        H, W = bgr.shape[:2]
        ids = np.zeros(MAXM, np.int32)
        corners = np.zeros((MAXM, 8), np.float32)
        conf = np.zeros(MAXM, np.float32)
        n = C.c_int(0)
        _lib.check(self.lib.fid_detect_with_confidence(self.h, bgr.ctypes.data_as(C.c_void_p), W, H, W * self.bpp, MAXM, C.byref(n), ids.ctypes.data_as(C.c_void_p),
                                                       corners.ctypes.data_as(C.c_void_p), conf.ctypes.data_as(C.c_void_p)), "fid_detect_with_confidence")
        return ids[: n.value].copy(), corners[: n.value].reshape(-1, 4, 2).copy(), conf[: n.value].copy()

    def set_marker_confidence(self, enable: bool):
        """fid_set_marker_confidence: batches submitted from now on also compute every marker's detection confidence."""
        _lib.check(self.lib.fid_set_marker_confidence(self.h, int(bool(enable))), "fid_set_marker_confidence")

    def last_marker_confidence(self, max_markers=MAXM):
        """fid_last_marker_confidence: float32 [n_frames, max_markers], laid out like the ids of the batch last returned."""
        nf = C.c_int(0)
        _lib.check(self.lib.fid_last_marker_confidence(self.h, max_markers, C.byref(nf), None), "fid_last_marker_confidence")
        out = np.zeros((nf.value, max_markers), np.float32)
        _lib.check(self.lib.fid_last_marker_confidence(self.h, max_markers, C.byref(nf), out.ctypes.data_as(C.c_void_p)), "fid_last_marker_confidence")
        return out

    def set_detect_inverted_marker(self, enable: bool):
        """fid_set_detect_inverted_marker (detectInvertedMarker): also detect white-on-black markers; a group of nested outlines then
        keeps its smallest, as in cv2, so black markers can come back with other corners."""
        _lib.check(self.lib.fid_set_detect_inverted_marker(self.h, int(bool(enable))), "fid_set_detect_inverted_marker")

    def set_aruco3(self, min_side: int = 32, ratio: float = 0.0, enable: bool = True):
        """fid_set_aruco3: useAruco3Detection with minSideLengthCanonicalImg = min_side and minMarkerLengthRatioOriginalImg = ratio
        (cv2's defaults 32 and 0); enable=False turns the mode off again."""
        p = _lib.fid_aruco3_params(int(bool(enable)), int(min_side), float(ratio))
        _lib.check(self.lib.fid_set_aruco3(self.h, C.byref(p)), "fid_set_aruco3")

    def debug_aruco3_planes(self, bgr):
        """fid_debug_aruco3_planes: (segmentation plane [seg_h, seg_w], [pyramid levels 1..], closest level) of one frame."""
        bgr = np.ascontiguousarray(bgr, np.uint8)
        H, W = bgr.shape[:2]
        info = np.zeros(4, np.int32)
        _lib.check(self.lib.fid_debug_aruco3_planes(self.h, bgr.ctypes.data_as(C.c_void_p), W, H, W * self.bpp, info.ctypes.data_as(C.c_void_p), None, None, 0),
                   "fid_debug_aruco3_planes")
        sw, sh, n_levels, closest = (int(v) for v in info)
        sizes, w, h = [], W, H
        for _ in range(n_levels - 1):
            w, h = (w + 1) // 2, (h + 1) // 2
            sizes.append((h, w))
        seg = np.zeros((sh, sw), np.uint8)
        pyr = np.zeros(max(1, sum(a * b for a, b in sizes)), np.uint8)
        _lib.check(self.lib.fid_debug_aruco3_planes(self.h, bgr.ctypes.data_as(C.c_void_p), W, H, W * self.bpp, info.ctypes.data_as(C.c_void_p),
                                                    seg.ctypes.data_as(C.c_void_p), pyr.ctypes.data_as(C.c_void_p), pyr.size), "fid_debug_aruco3_planes")
        levels, off = [], 0
        for h, w in sizes:
            levels.append(pyr[off:off + h * w].reshape(h, w).copy())
            off += h * w
        return seg, levels, closest

    def set_pose_hypotheses(self, enable: bool):
        """fid_set_pose_hypotheses: batches submitted from now on also compute both planar pose solutions of every marker."""
        _lib.check(self.lib.fid_set_pose_hypotheses(self.h, int(bool(enable))), "fid_set_pose_hypotheses")

    def pose_hypotheses(self, ids, corners, K, D, fiducial_len, overrides: Optional[Dict[int, float]] = None):
        """fid_pose_hypotheses: both IPPE_SQUARE solutions of markers already detected (arguments as pose())."""
        ids = np.ascontiguousarray(ids, np.int32)
        corners = np.ascontiguousarray(corners, np.float32).reshape(-1, 8)
        n = len(ids)
        out = (_lib.fid_pose_hypotheses * max(n, 1))()
        cam = _camera(K, D)
        oi, ol, no = _overrides(overrides)
        _lib.check(self.lib.fid_pose_hypotheses(self.h, n, ids.ctypes.data_as(C.c_void_p), corners.ctypes.data_as(C.c_void_p), C.byref(cam), float(fiducial_len), no,
                                                oi.ctypes.data_as(C.c_void_p), ol.ctypes.data_as(C.c_void_p), C.cast(out, C.c_void_p)), "fid_pose_hypotheses")
        return [out[i] for i in range(n)]

    def last_pose_hypotheses(self, max_markers=MAXM):
        """fid_last_pose_hypotheses: records of the batch last returned by detect_pose_batch / collect_batch, as a ctypes array
        [n_frames * max_markers] laid out like its transforms (record f * max_markers + m belongs to marker m of frame f)."""
        nf = C.c_int(0)
        _lib.check(self.lib.fid_last_pose_hypotheses(self.h, max_markers, C.byref(nf), None), "fid_last_pose_hypotheses")
        out = (_lib.fid_pose_hypotheses * max(nf.value * max_markers, 1))()
        _lib.check(self.lib.fid_last_pose_hypotheses(self.h, max_markers, C.byref(nf), C.cast(out, C.c_void_p)), "fid_last_pose_hypotheses")
        return out

    @staticmethod
    def _families(families, n):
        fam = np.ascontiguousarray(families, np.int32).reshape(-1)
        if len(fam) != n:
            raise ValueError("one family per board: %d boards, %d families" % (n, len(fam)))
        return fam

    def set_boards(self, boards, families=None):
        """fid_set_boards: a list of fiducials_b200.board.Board (empty = off).  Batches submitted with a camera from now on also
        solve one pose per (frame, board).  families: one dictionary index per board (fid_set_family_boards), which a
        multi-dictionary handle needs; None leaves the boards without a family."""
        boards = list(boards)
        keep = [(np.ascontiguousarray(b.ids, np.int32), np.ascontiguousarray(b.obj_points, np.float32)) for b in boards]
        arr = (_lib.fid_board * max(len(keep), 1))()
        for i, (ids, obj) in enumerate(keep):
            arr[i].n_markers = len(ids)
            arr[i].ids = ids.ctypes.data
            arr[i].obj_points = obj.ctypes.data
        if families is None:
            _lib.check(self.lib.fid_set_boards(self.h, len(keep), C.cast(arr, C.c_void_p)), "fid_set_boards")
        else:
            fam = self._families(families, len(keep))
            _lib.check(self.lib.fid_set_family_boards(self.h, len(keep), C.cast(arr, C.c_void_p), fam.ctypes.data_as(C.c_void_p)), "fid_set_family_boards")
        self.n_boards = len(keep)

    def board_poses(self, ids, corners, K, D):
        """fid_estimate_board_poses: one fid_board_pose per board set, for markers already detected (ids, corners as detect())."""
        ids = np.ascontiguousarray(ids, np.int32).reshape(-1)
        corners = np.ascontiguousarray(corners, np.float32).reshape(-1, 8)
        nb = getattr(self, "n_boards", 0)
        out = (_lib.fid_board_pose * max(nb, 1))()
        cam = _camera(K, D)
        _lib.check(self.lib.fid_estimate_board_poses(self.h, len(ids), ids.ctypes.data_as(C.c_void_p), corners.ctypes.data_as(C.c_void_p), C.byref(cam),
                                                     C.cast(out, C.c_void_p)), "fid_estimate_board_poses")
        return [out[i] for i in range(nb)]

    def last_board_poses(self):
        """fid_last_board_poses: records of the batch last returned by detect_pose_batch / collect_batch, a list per frame of
        one fid_board_pose per board."""
        nf, nb = C.c_int(0), C.c_int(0)
        _lib.check(self.lib.fid_last_board_poses(self.h, 0, C.byref(nf), C.byref(nb), None), "fid_last_board_poses")
        out = (_lib.fid_board_pose * max(nf.value * nb.value, 1))()
        _lib.check(self.lib.fid_last_board_poses(self.h, nb.value, C.byref(nf), C.byref(nb), C.cast(out, C.c_void_p)), "fid_last_board_poses")
        return [[out[f * nb.value + b] for b in range(nb.value)] for f in range(nf.value)]

    def set_charuco_boards(self, boards, families=None):
        """fid_set_charuco_boards: a list of fiducials_b200.board.CharucoBoard (empty = off).  Batches submitted from now on also
        find each board's chessboard corners (and, with a camera, its pose).  families: as set_boards
        (fid_set_family_charuco_boards)."""
        boards = list(boards)
        arr = (_lib.fid_charuco_board * max(len(boards), 1))()
        keep = []
        for i, b in enumerate(boards):
            ids = np.ascontiguousarray(b.ids, np.int32)
            keep.append(ids)
            arr[i].squares_x, arr[i].squares_y = b.size
            arr[i].square_length, arr[i].marker_length = b.square_length, b.marker_length
            arr[i].legacy_pattern, arr[i].ids = int(b.legacy), ids.ctypes.data
            arr[i].min_markers, arr[i].check_markers = b.min_markers, int(b.check_markers)
        if families is None:
            _lib.check(self.lib.fid_set_charuco_boards(self.h, len(boards), C.cast(arr, C.c_void_p)), "fid_set_charuco_boards")
        else:
            fam = self._families(families, len(boards))
            _lib.check(self.lib.fid_set_family_charuco_boards(self.h, len(boards), C.cast(arr, C.c_void_p), fam.ctypes.data_as(C.c_void_p)),
                       "fid_set_family_charuco_boards")
        self.charuco_boards = boards

    def _charuco_split(self, recs, cids, cxy):
        out = []
        for r in recs:
            o, n = int(r.corner_offset), int(r.n_corners)
            out.append((r, cids[o:o + n].copy(), cxy[o:o + n].copy()))
        return out

    def charuco(self, frame, ids, corners, K=None, D=None):
        """fid_detect_charuco: per ChArUco board set, (fid_charuco_result, corner ids [n], corners [n, 2]) for one frame and markers
        already detected (ids, corners as detect()).  Without K no pose."""
        frame = np.ascontiguousarray(frame, np.uint8)
        H, W = frame.shape[:2]
        ids = np.ascontiguousarray(ids, np.int32).reshape(-1)
        corners = np.ascontiguousarray(corners, np.float32).reshape(-1, 8)
        boards = getattr(self, "charuco_boards", [])
        slots = sum(b.n_corners for b in boards)
        recs = (_lib.fid_charuco_result * max(len(boards), 1))()
        cids = np.zeros(max(slots, 1), np.int32)
        cxy = np.zeros((max(slots, 1), 2), np.float32)
        cam = None if K is None else C.byref(_camera(K, D))
        _lib.check(self.lib.fid_detect_charuco(self.h, frame.ctypes.data_as(C.c_void_p), W, H, frame.strides[0], len(ids), ids.ctypes.data_as(C.c_void_p),
                                               corners.ctypes.data_as(C.c_void_p), cam, C.cast(recs, C.c_void_p), cids.ctypes.data_as(C.c_void_p),
                                               cxy.ctypes.data_as(C.c_void_p)), "fid_detect_charuco")
        return self._charuco_split([recs[i] for i in range(len(boards))], cids, cxy)

    def last_charuco(self):
        """fid_last_charuco: for the batch last returned by detect_pose_batch / collect_batch, a list per frame of
        (fid_charuco_result, corner ids, corners) per ChArUco board."""
        nf, nb, ns = C.c_int(0), C.c_int(0), C.c_int(0)
        _lib.check(self.lib.fid_last_charuco(self.h, 0, C.byref(nf), C.byref(nb), C.byref(ns), None, None, None), "fid_last_charuco")
        recs = (_lib.fid_charuco_result * max(nf.value * nb.value, 1))()
        cids = np.zeros((max(nf.value, 1), max(ns.value, 1)), np.int32)
        cxy = np.zeros((max(nf.value, 1), max(ns.value, 1), 2), np.float32)
        _lib.check(self.lib.fid_last_charuco(self.h, cids.shape[1], C.byref(nf), C.byref(nb), C.byref(ns), C.cast(recs, C.c_void_p), cids.ctypes.data_as(C.c_void_p),
                                             cxy.ctypes.data_as(C.c_void_p)), "fid_last_charuco")
        return [self._charuco_split([recs[f * nb.value + b] for b in range(nb.value)], cids[f], cxy[f]) for f in range(nf.value)]

    def set_marker_refinement(self, min_rep_distance=10.0, error_correction_rate=3.0, check_all_orders=True):
        """fid_set_marker_refinement: cv::aruco::RefineParameters for refine_markers (min_rep_distance=None turns it off)."""
        p = _lib.fid_marker_refine_params()
        if min_rep_distance is not None:
            p.enable, p.min_rep_distance, p.error_correction_rate, p.check_all_orders = 1, min_rep_distance, error_correction_rate, int(bool(check_all_orders))
        _lib.check(self.lib.fid_set_marker_refinement(self.h, C.byref(p)), "fid_set_marker_refinement")

    def refine_markers(self, frame, ids, corners, rejected, K=None, D=None):
        """fid_refine_detected_markers: cv2.aruco.ArucoDetector.refineDetectedMarkers against every marker board and then every
        ChArUco board set, for one frame and the lists of its detection (ids [n], corners [n, 4, 2], rejected [m, 4, 2]).  Returns
        what cv2 returns: ids, corners, the rejected candidates left, and recovered_idx (indices into `rejected`), plus the board of
        each recovered marker (b for marker board b, FID_MAX_BOARDS + c for ChArUco board c)."""
        frame = np.ascontiguousarray(frame, np.uint8)
        H, W = frame.shape[:2]
        ids = np.ascontiguousarray(ids, np.int32).reshape(-1)
        n = len(ids)
        oi = np.zeros(MAXM, np.int32)
        oc = np.zeros((MAXM, 8), np.float32)
        oi[:n] = ids
        oc[:n] = np.asarray(corners, np.float32).reshape(-1, 8)
        rej = np.ascontiguousarray(np.asarray(rejected, np.float32).reshape(-1, 8))
        ri, rb = np.zeros(MAXM, np.int32), np.zeros(MAXM, np.int32)
        nout = C.c_int(0)
        cam = None if K is None else C.byref(_camera(K, D))
        _lib.check(self.lib.fid_refine_detected_markers(self.h, frame.ctypes.data_as(C.c_void_p), W, H, frame.strides[0], n, oi.ctypes.data_as(C.c_void_p),
                                                        oc.ctypes.data_as(C.c_void_p), MAXM, len(rej), rej.ctypes.data_as(C.c_void_p), cam, C.byref(nout),
                                                        ri.ctypes.data_as(C.c_void_p), rb.ctypes.data_as(C.c_void_p)), "fid_refine_detected_markers")
        nr = nout.value - n
        taken = set(ri[:nr].tolist())
        left = np.array([r for k, r in enumerate(rej) if k not in taken], np.float32).reshape(-1, 4, 2)
        return oi[: nout.value].copy(), oc[: nout.value].reshape(-1, 4, 2).copy(), left, ri[:nr].copy(), rb[:nr].copy()

    def set_batch_marker_refinement(self, enable: bool):
        """fid_set_batch_marker_refinement: batches submitted from now on recover missed board markers (with set_marker_refinement
        enabled and a board set); the recovered markers are appended to each frame's markers."""
        _lib.check(self.lib.fid_set_batch_marker_refinement(self.h, int(bool(enable))), "fid_set_batch_marker_refinement")

    def last_marker_refinement(self):
        """fid_last_marker_refinement: for the batch last returned by detect_pose_batch / collect_batch, a list per frame of
        (recovered_idx, recovered_board, rejected before refinement [m, 4, 2], rejected left [m - n_recovered, 4, 2]) -- the last two
        as cv2's detectMarkers and refineDetectedMarkers return rejectedImgPoints.  The recovered markers are the frame's last
        len(recovered_idx) markers."""
        nf = C.c_int(0)
        _lib.check(self.lib.fid_last_marker_refinement(self.h, 0, 0, C.byref(nf), None, None, None, None, None), "fid_last_marker_refinement")
        n = max(nf.value, 1)
        nrec, nrej = np.zeros(n, np.int32), np.zeros(n, np.int32)
        _lib.check(self.lib.fid_last_marker_refinement(self.h, 0, 0, C.byref(nf), nrec.ctypes.data_as(C.c_void_p), None, None, nrej.ctypes.data_as(C.c_void_p), None),
                   "fid_last_marker_refinement")
        mm, mj = max(int(nrec.max()), 1), max(int(nrej.max()), 1)
        ri, rb = np.zeros((n, mm), np.int32), np.zeros((n, mm), np.int32)
        rej = np.zeros((n, mj, 8), np.float32)
        _lib.check(self.lib.fid_last_marker_refinement(self.h, mm, mj, C.byref(nf), None, ri.ctypes.data_as(C.c_void_p), rb.ctypes.data_as(C.c_void_p), None,
                                                       rej.ctypes.data_as(C.c_void_p)), "fid_last_marker_refinement")
        out = []
        for f in range(nf.value):
            r, j = int(nrec[f]), int(nrej[f])
            before = rej[f, :j].reshape(-1, 4, 2).copy()
            taken = set(ri[f, :r].tolist())
            left = np.array([q for k, q in enumerate(before) if k not in taken], np.float32).reshape(-1, 4, 2)
            out.append((ri[f, :r].copy(), rb[f, :r].copy(), before, left))
        return out

    def set_diamonds(self, square_length, marker_length=None, min_markers=2, check_markers=True, family=None):
        """fid_set_diamonds: the ChArUco diamond geometry (square_length=None turns diamonds off).  Batches submitted from now on also
        find each frame's diamonds (and, with a camera, their poses).  family: the dictionary index of the diamonds' markers
        (fid_set_family_diamonds), which a multi-dictionary handle needs; None sets them without a family."""
        p = _lib.fid_diamond_params()
        if square_length is not None:
            p.enable, p.square_length, p.marker_length = 1, square_length, marker_length
            p.min_markers, p.check_markers = int(min_markers), int(bool(check_markers))
        if family is None:
            _lib.check(self.lib.fid_set_diamonds(self.h, C.byref(p)), "fid_set_diamonds")
        else:
            _lib.check(self.lib.fid_set_family_diamonds(self.h, C.byref(p), int(family)), "fid_set_family_diamonds")

    @staticmethod
    def _diamond_split(recs):
        """(ids [k, 4] int32, corners [k, 4, 2] float32, fid_diamond records) -- cv2's diamondIds and diamondCorners, and the poses."""
        ids = np.array([list(r.ids) for r in recs], np.int32).reshape(-1, 4)
        corners = np.array([list(r.corners) for r in recs], np.float32).reshape(-1, 4, 2)
        return ids, corners, list(recs)

    def diamonds(self, frame, ids, corners, K=None, D=None):
        """fid_detect_diamonds: the diamonds of one frame among markers already detected (ids, corners as detect()), as
        cv2.aruco.CharucoDetector.detectDiamonds finds them.  Without K no pose.  Returns (ids, corners, records)."""
        frame = np.ascontiguousarray(frame, np.uint8)
        H, W = frame.shape[:2]
        ids = np.ascontiguousarray(ids, np.int32).reshape(-1)
        corners = np.ascontiguousarray(corners, np.float32).reshape(-1, 8)
        out = (_lib.fid_diamond * max(len(ids) // 4, 1))()
        nd = C.c_int(0)
        cam = None if K is None else C.byref(_camera(K, D))
        _lib.check(self.lib.fid_detect_diamonds(self.h, frame.ctypes.data_as(C.c_void_p), W, H, frame.strides[0], len(ids), ids.ctypes.data_as(C.c_void_p),
                                                corners.ctypes.data_as(C.c_void_p), cam, C.byref(nd), C.cast(out, C.c_void_p)), "fid_detect_diamonds")
        return self._diamond_split([out[i] for i in range(nd.value)])

    def last_diamonds(self):
        """fid_last_diamonds: for the batch last returned by detect_pose_batch / collect_batch, a list per frame of (ids, corners,
        records) as diamonds() returns them."""
        nf = C.c_int(0)
        _lib.check(self.lib.fid_last_diamonds(self.h, 0, C.byref(nf), None, None), "fid_last_diamonds")
        counts = np.zeros(max(nf.value, 1), np.int32)
        _lib.check(self.lib.fid_last_diamonds(self.h, 0, C.byref(nf), counts.ctypes.data_as(C.c_void_p), None), "fid_last_diamonds")
        m = max(int(counts.max()), 1)
        out = (_lib.fid_diamond * (max(nf.value, 1) * m))()
        _lib.check(self.lib.fid_last_diamonds(self.h, m, C.byref(nf), None, C.cast(out, C.c_void_p)), "fid_last_diamonds")
        return [self._diamond_split([out[f * m + k] for k in range(int(counts[f]))]) for f in range(nf.value)]

    def debug_rejected(self):
        """fid_debug_rejected: detectMarkers' rejectedImgPoints [m, 4, 2] for the last detect() call."""
        n = C.c_int(0)
        out = np.zeros((_lib.FID_MAX_REJECTED, 8), np.float32)
        _lib.check(self.lib.fid_debug_rejected(self.h, len(out), C.byref(n), out.ctypes.data_as(C.c_void_p)), "fid_debug_rejected")
        return out[: n.value].reshape(-1, 4, 2).copy()

    def debug_threshold(self, bgr):
        bgr = np.ascontiguousarray(bgr, np.uint8)
        H, W = bgr.shape[:2]
        gray = np.zeros((H, W), np.uint8)
        planes = np.zeros((16, H, W), np.uint8)
        ns = C.c_int(0)
        _lib.check(self.lib.fid_debug_threshold(self.h, bgr.ctypes.data_as(C.c_void_p), W, H, W * self.bpp, gray.ctypes.data_as(C.c_void_p), planes.ctypes.data_as(C.c_void_p),
                                                C.byref(ns)))
        return gray, planes[: ns.value]

    def debug_candidates(self):
        cap = 4096
        quads = np.zeros((cap, 8), np.int32)
        scale = np.zeros(cap, np.int32)
        clen = np.zeros(cap, np.int32)
        n = C.c_int(0)
        _lib.check(self.lib.fid_debug_candidates(self.h, cap, C.byref(n), quads.ctypes.data_as(C.c_void_p), scale.ctypes.data_as(C.c_void_p),
                                                 clen.ctypes.data_as(C.c_void_p)))
        return quads[: n.value].reshape(-1, 4, 2), scale[: n.value], clen[: n.value]

    STAGES = ["h2d", "threshold", "masks_starts", "walk", "emit", "approx", "group", "identify", "subpix_pose", "_", "d2h", "walk_r0", "walk_r1", "walk_r2", "walk_r3", "walk_r4", "walk_r5", "walk_r6", "walk_r7"]

    def last_stage_ms(self):
        ms = np.zeros(32, np.float32)
        n = C.c_int(0)
        _lib.check(self.lib.fid_last_stage_ms(self.h, ms.ctypes.data_as(C.c_void_p), 32, C.byref(n)))
        return {k: float(ms[i]) for i, k in enumerate(self.STAGES) if k != "_"}

    COUNTERS = ["start_cracks", "contours_in_range", "contour_points", "quad_candidates", "selected", "markers", "kernel_launches"]

    def last_counters(self):
        c = np.zeros(8, np.int64)
        n = C.c_int(0)
        _lib.check(self.lib.fid_last_counters(self.h, c.ctypes.data_as(C.c_void_p), 8, C.byref(n)))
        return {k: int(c[i]) for i, k in enumerate(self.COUNTERS)}


def _overrides(overrides):
    if not overrides:
        return np.zeros(1, np.int32), np.zeros(1, np.float64), 0
    ks = sorted(overrides)
    return np.array(ks, np.int32), np.array([overrides[k] for k in ks], np.float64), len(ks)


class FiducialsNode:
    """aruco_detect's node, minus ROS transport."""

    def __init__(self, dictionary=7, fiducial_len=0.14, ignore_fiducials: Iterable[int] = (), fiducial_len_override: Optional[Dict[int, float]] = None,
                 do_pose_estimation=True, device=0, max_width=1920, max_height=1080, max_batch=1, doCornerRefinement=True, cornerRefinementSubPix=True, pose_hypotheses=False,
                 boards=(), charuco_boards=(), refine_markers=None, diamonds=None, dictionaries=(), aruco3=None, detect_inverted_marker=False,
                 **detector_params):
        # doCornerRefinement / cornerRefinementSubPix -> cornerRefinementMethod NONE / SUBPIX / CONTOUR (:700-711, configCallback :274-281)
        if refine_markers is not None and not boards and not charuco_boards:
            raise ValueError("refine_markers needs boards or charuco_boards")
        detector_params.setdefault("cornerRefinementMethod", (1 if cornerRefinementSubPix else 2) if doCornerRefinement else 0)
        self.fiducial_len = float(fiducial_len)  # :615
        self.doPoseEstimation = do_pose_estimation  # :614
        self.ignoreIds = set(int(i) for i in ignore_fiducials)  # :540-571
        self.fiducialLens = dict(fiducial_len_override or {})  # :627-660
        self.det = Detector(default_params(dictionary=dictionary, **detector_params), device, max_width, max_height, max_batch)
        # further dictionaries (new, no reference counterpart): dictionaries = [(dictionary, id_offset, fiducial_len), ...] after
        # `dictionary`; detection is detectMarkersMultiDict, the messages carry published ids (id + id_offset), and ignore_fiducials /
        # fiducial_len_override are keyed by them; a dictionary's fiducial_len of 0 means fiducial_len
        self.dictSpecs = [(int(dictionary), 0, 0.0)] + [(int(d), int(o), float(l)) for d, o, l in dictionaries]
        if len(self.dictSpecs) > 1:
            self.det.set_dictionaries(self.dictSpecs)
        self.dictIdx = np.zeros(0, np.int32)
        # detection on a downscaled frame (new, no reference counterpart): aruco3 = (minMarkerLengthRatioOriginalImg,
        # minSideLengthCanonicalImg) turns on cv2's useAruco3Detection; the messages carry the full-resolution corners it returns
        if aruco3 is not None:
            self.det.set_aruco3(int(aruco3[1]), float(aruco3[0]))
        # white-on-black markers too (new, no reference counterpart): cv2's detectInvertedMarker; a group of nested outlines then keeps
        # its smallest, so black markers come back with cv2's corners under the flag, not the reference's
        if detect_inverted_marker:
            self.det.set_detect_inverted_marker(True)
        # both planar pose solutions of every marker (new, no reference counterpart): when on, the pose results carry an extra
        # attribute `pose_hypotheses` = {fiducial_id: fid_pose_hypotheses record}; their message fields are unchanged
        self.poseHypotheses = bool(pose_hypotheses)
        if self.poseHypotheses:
            self.det.set_pose_hypotheses(True)
        # one pose per marker board (new, no reference counterpart): with boards (fiducials_b200.board.Board) the pose results carry
        # an extra attribute `board_poses` = [fid_board_pose record per board, in board order]; their message fields are unchanged
        # with `dictionaries`, an entry may be (board, family): the board's markers are those of that entry of the node's list (0 =
        # `dictionary`), which a multi-dictionary node needs for every board, ChArUco board and the diamonds
        self.boards, families = _with_families(boards)
        if self.boards:
            self.det.set_boards(self.boards, families)
        # ChArUco boards (new, no reference counterpart): with charuco_boards (fiducials_b200.board.CharucoBoard) the pose results
        # carry an extra attribute `charuco` = [(fid_charuco_result, corner ids, corners [n, 2]) per board, in board order]
        self.charucoBoards, families = _with_families(charuco_boards)
        if self.charucoBoards:
            self.det.set_charuco_boards(self.charucoBoards, families)
        # recovery of missed board markers (new, no reference counterpart): refine_markers = (min_rep_distance, error_correction_rate,
        # check_all_orders) runs cv2's refineDetectedMarkers against the boards after detection; the recovered markers are reported
        # like any other marker, and the results carry `recovered` = [(fiducial_id, board)] (board b, or FID_MAX_BOARDS + c for
        # ChArUco board c)
        self.refineMarkers = refine_markers is not None
        if self.refineMarkers:
            self.det.set_marker_refinement(*refine_markers)
            self.det.set_batch_marker_refinement(True)
        # ChArUco diamonds (new, no reference counterpart): diamonds = (square_length, marker_length) finds cv2's detectDiamonds among
        # the markers; the pose results carry `diamonds` = (ids [k, 4], corners [k, 4, 2], fid_diamond records with the poses);
        # (square_length, marker_length, family) binds them to a family as the boards above
        self.diamondGeometry = diamonds
        if diamonds is not None:
            self.det.set_diamonds(diamonds[0], diamonds[1], family=diamonds[2] if len(diamonds) > 2 else None)
        # with several dictionaries the board stages read each family's markers in the one-frame batch (the stand-alone calls take
        # lists without a family); poseEstimateCallback then publishes that batch's records
        self._batchStages = len(self.dictSpecs) > 1 and bool(self.boards or self.charucoBoards or diamonds is not None)
        self._stageRecords = (None, None, None)
        self._recovered = []
        self._last_frame = None  # the frame of the last imageCallback, for the ChArUco corners of poseEstimateCallback
        self.haveCamInfo = False
        self.K = None
        self.D = None
        self.frameId = ""
        self.frameNum = 0
        self.enable_detections = True
        self.vis_msgs = False  # pnh.param vis_msgs (:614)
        self.ids = np.zeros(0, np.int32)
        self.corners = np.zeros((0, 4, 2), np.float32)
        self._last_header = Header()

    # :307-330
    def camInfoCallback(self, K, D, frame_id=""):
        if self.haveCamInfo:
            return
        K = np.asarray(K, np.float64).reshape(3, 3)
        if np.all(K == 0.0):  # :313 "CameraInfo message has invalid intrinsics, K matrix all zeros"
            return
        self.K = K
        self.D = np.asarray(D, np.float64).reshape(-1)[:5]
        self.haveCamInfo = True
        self.frameId = frame_id

    # :332-395
    def imageCallback(self, bgr, header: Optional[Header] = None) -> Optional[FiducialArray]:
        if not self.enable_detections:
            return None  # :334
        header = header or Header()
        fva = FiducialArray(header=Header(header.seq, header.stamp, self.frameId))
        try:
            if self.refineMarkers:  # the one-frame batch, which refines (detect() is detectMarkers alone)
                counts, ids, corners, _ = self.det.detect_pose_batch(np.ascontiguousarray(bgr, np.uint8)[None])
                n = int(counts[0])
                self.ids, self.corners = ids[0, :n].copy(), corners[0, :n].copy()
                idx, brd, _, _ = self.det.last_marker_refinement()[0]
                self._recovered = self._recovered_of(self.ids, idx, brd)
            elif self._batchStages:
                cam = (self.K, self.D, self.fiducial_len, self.fiducialLens) if self.haveCamInfo and self.doPoseEstimation else ()
                counts, ids, corners, _ = self.det.detect_pose_batch(np.ascontiguousarray(bgr, np.uint8)[None], *cam)
                n = int(counts[0])
                self.ids, self.corners = ids[0, :n].copy(), corners[0, :n].copy()
                self.dictIdx = self.det.last_dict_indices()[0, :n].copy()
                self._stageRecords = (self.det.last_board_poses()[0] if self.boards and cam else None,
                                      self.det.last_charuco()[0] if self.charucoBoards else None,
                                      self.det.last_diamonds()[0] if self.diamondGeometry is not None else None)
            elif len(self.dictSpecs) > 1:
                self.ids, self.corners, self.dictIdx = self.det.detect_multi_dict(bgr)
            else:
                self.ids, self.corners = self.det.detect(bgr)  # :350
        except _lib.FidError:
            return None  # frame dropped (:389-394)
        if len(self.dictSpecs) == 1:
            self.dictIdx = np.zeros(len(self.ids), np.int32)
        if self.charucoBoards or self.diamondGeometry is not None:
            self._last_frame = np.ascontiguousarray(bgr, np.uint8)
        for i, fid in enumerate(self._published().tolist()):
            if fid in self.ignoreIds:
                continue  # :359-364
            c = self.corners[i]
            fva.fiducials.append(Fiducial(fid, 0, *[float(v) for v in c.reshape(-1)]))  # :366-376
        if self.refineMarkers:
            fva.recovered = self._recovered
        self._last_header = header
        return fva

    def _published(self):
        """The published ids of the last imageCallback's markers: id + their dictionary's id_offset."""
        offsets = np.array([s[1] for s in self.dictSpecs], np.int32)
        return self.ids + offsets[self.dictIdx]

    def _per_dictionary(self, solve):
        """solve(published ids, corners, length) once per dictionary over its markers; the records in marker order."""
        if len(self.dictSpecs) == 1:
            return solve(self.ids, self.corners, self.fiducial_len)
        out = [None] * len(self.ids)
        pub = self._published()
        for d, (_, _, ln) in enumerate(self.dictSpecs):
            sel = np.where(self.dictIdx == d)[0]
            if len(sel):
                for m, r in zip(sel.tolist(), solve(pub[sel], self.corners[sel], ln if ln > 0 else self.fiducial_len)):
                    out[m] = r
        return out

    def _recovered_of(self, ids, idx, boards):
        """The frame's recovered markers (its last len(idx) markers) as (fiducial_id, board), without the ignored ids."""
        n0 = len(ids) - len(idx)
        return [(int(i), int(b)) for i, b in zip(ids[n0:].tolist(), boards.tolist()) if i not in self.ignoreIds]

    # :397-538
    def poseEstimateCallback(self, msg: Optional[FiducialArray] = None) -> Optional[FiducialTransformArray]:
        header = msg.header if msg is not None else self._last_header
        fta = FiducialTransformArray(header=Header(0, header.stamp, self.frameId), image_seq=header.seq)
        self.frameNum += 1
        if not self.doPoseEstimation:
            return fta
        if not self.haveCamInfo:
            return None  # :417-422
        try:
            tfs = self._per_dictionary(lambda i, c, ln: self.det.pose(i, c, self.K, self.D, ln, self.fiducialLens))
            hyps = self._per_dictionary(lambda i, c, ln: self.det.pose_hypotheses(i, c, self.K, self.D, ln, self.fiducialLens)) if self.poseHypotheses else None
            if self._batchStages:
                boards, charuco, diamonds = self._stageRecords
            else:
                boards = self.det.board_poses(self.ids, self.corners, self.K, self.D) if self.boards else None
                charuco = self.det.charuco(self._last_frame, self.ids, self.corners, self.K, self.D) if self.charucoBoards and self._last_frame is not None else None
                diamonds = self.det.diamonds(self._last_frame, self.ids, self.corners, self.K, self.D) if self.diamondGeometry is not None and self._last_frame is not None else None
        except _lib.FidError:
            return fta
        if self.vis_msgs:  # :403, :462-478: vision_msgs/Detection2DArray instead of FiducialTransformArray
            vma = Detection2DArray(header=Header(0, header.stamp, self.frameId))
            for t in tfs:
                if t.fiducial_id in self.ignoreIds:
                    continue
                vma.detections.append(Detection2D([ObjectHypothesisWithPose(int(t.fiducial_id), math.exp(-2.0 * float(t.object_error)), tuple(t.translation), tuple(t.rotation))]))
            if hyps is not None:
                vma.pose_hypotheses = self._by_id(hyps)
            if boards is not None:
                vma.board_poses = boards
            if charuco is not None:
                vma.charuco = charuco
            if diamonds is not None:
                vma.diamonds = diamonds
            if self.refineMarkers:
                vma.recovered = self._recovered
            return vma
        for t in tfs:
            if t.fiducial_id in self.ignoreIds:
                continue  # :440
            fta.transforms.append(_to_msg(t))
        if hyps is not None:
            fta.pose_hypotheses = self._by_id(hyps)
        if boards is not None:
            fta.board_poses = boards
        if charuco is not None:
            fta.charuco = charuco
        if diamonds is not None:
            fta.diamonds = diamonds
        if self.refineMarkers:
            fta.recovered = self._recovered
        return fta

    def _by_id(self, records):
        return {int(r.fiducial_id): r for r in records if r.fiducial_id not in self.ignoreIds}

    def process_batch(self, frames, first_seq=0) -> List[FiducialTransformArray]:
        """Throughput path: detect + pose for a stack of frames in one C-ABI call."""
        if not self.haveCamInfo:
            return []
        counts, ids, corners, tfs = self.det.detect_pose_batch(frames, self.K, self.D, self.fiducial_len, self.fiducialLens)
        hyps = self.det.last_pose_hypotheses() if self.poseHypotheses else None
        boards = self.det.last_board_poses() if self.boards else None
        charuco = self.det.last_charuco() if self.charucoBoards else None
        refined = self.det.last_marker_refinement() if self.refineMarkers else None
        diamonds = self.det.last_diamonds() if self.diamondGeometry is not None else None
        out = []
        for f in range(len(counts)):
            fta = FiducialTransformArray(header=Header(0, (0, 0), self.frameId), image_seq=first_seq + f)
            for m in range(int(counts[f])):
                t = tfs[f * MAXM + m]
                if t.fiducial_id not in self.ignoreIds:
                    fta.transforms.append(_to_msg(t))
            if hyps is not None:
                fta.pose_hypotheses = self._by_id(hyps[f * MAXM + m] for m in range(int(counts[f])))
            if boards is not None:
                fta.board_poses = boards[f]
            if charuco is not None:
                fta.charuco = charuco[f]
            if diamonds is not None:
                fta.diamonds = diamonds[f]
            if refined is not None:
                fta.recovered = self._recovered_of(ids[f, : int(counts[f])], refined[f][0], refined[f][1])
            out.append(fta)
        return out


def _with_families(items):
    """Boards given as board or (board, family): (boards, families), families None when no entry names one (the setters without a
    family), else one per board with 0 for a bare board."""
    items = list(items)
    if not any(isinstance(b, tuple) for b in items):
        return items, None
    pairs = [b if isinstance(b, tuple) else (b, 0) for b in items]
    return [b for b, _ in pairs], [int(f) for _, f in pairs]


def _to_msg(t) -> FiducialTransform:
    return FiducialTransform(int(t.fiducial_id), Transform(tuple(t.translation), tuple(t.rotation)), float(t.image_error), float(t.object_error), float(t.fiducial_area))


def _tf(T) -> Optional["_lib.fid_tf"]:
    if T is None:
        return None
    t = _lib.fid_tf()
    for i in range(3):
        t.t[i] = float(T[i])
    for i in range(4):
        t.q[i] = float(T[3 + i])
    return t


class FiducialSlam:
    """fiducial_slam's node, minus ROS transport: transformCallback + Map state on the device."""

    def __init__(self, device=0, max_fiducials=512, n_instances=1, weighting_scale=1e9, use_fiducial_area_as_weight=False, read_only_map=False):
        self.lib = _lib.load()
        p = _lib.fid_map_params()
        _lib.check(self.lib.fid_map_default_params(C.byref(p)))
        p.max_fiducials = max_fiducials
        p.n_instances = n_instances
        p.weighting_scale = weighting_scale
        p.use_fiducial_area_as_weight = int(use_fiducial_area_as_weight)
        p.read_only_map = int(read_only_map)
        self.p = p
        self.h = C.c_void_p()
        _lib.check(self.lib.fid_map_create(C.byref(p), device, C.byref(self.h)), "fid_map_create")

    def close(self):
        if getattr(self, "h", None) is not None and self.h.value:
            self.lib.fid_map_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def loadMap(self, entries: Sequence[Sequence[float]], instance=0):
        """entries: rows of the map file: id x y z roll pitch yaw(deg) variance numObs (map.cpp:556-562)."""
        arr = (_lib.fid_map_file_entry * len(entries))()
        for i, e in enumerate(entries):
            arr[i].fiducial_id = int(e[0])
            arr[i].x, arr[i].y, arr[i].z, arr[i].roll_deg, arr[i].pitch_deg, arr[i].yaw_deg, arr[i].variance = [float(v) for v in e[1:8]]
            arr[i].num_obs = int(e[8]) if len(e) > 8 else 0
        _lib.check(self.lib.fid_map_load(self.h, instance, len(entries), C.cast(arr, C.c_void_p)))

    def links(self, instance=0):
        """fid_map_links: {fiducial_id: sorted linked ids} (Fiducial::links, map.h:87)."""
        cap = self.p.max_fiducials
        pairs = np.zeros((cap * cap, 2), np.int32)
        n = C.c_int(0)
        _lib.check(self.lib.fid_map_links(self.h, instance, cap * cap, C.byref(n), pairs.ctypes.data_as(C.c_void_p)))
        out: Dict[int, List[int]] = {}
        for a, b in pairs[: n.value]:
            out.setdefault(int(a), []).append(int(b))
        return out

    def saveMap(self, filename, instance=0):
        """Map::saveMap, map.cpp:541-566: `id x y z rx ry rz(deg) variance numObs links...`, %lf formatting."""
        links = self.links(instance)
        with open(filename, "w") as fp:
            for e in self.entries(instance):
                rad2deg = lambda a: a * 180.0 / math.pi  # helpers.h:8
                fp.write("%d %f %f %f %f %f %f %f %d" % (e.fiducial_id, e.x, e.y, e.z, rad2deg(e.rx), rad2deg(e.ry), rad2deg(e.rz), e.variance, e.num_obs))
                fp.write("".join(" %d" % k for k in links.get(e.fiducial_id, [])) + "\n")
        return True

    def loadMapFile(self, filename, instance=0):
        """Map::loadMap(filename), map.cpp:572-625.  Returns the number of entries read (invalid lines are skipped
        like the reference's ROS_WARN("Invalid line"))."""
        rows, pairs = [], []
        with open(filename) as fp:
            for line in fp:
                # sscanf("%d %lf ... %d%[^\t\n]"): nine numbers separated by any white space (tabs too), then the links up to a tab
                m = re.match(r"\s*(\S+)\s+(\S+)\s+(\S+)\s+(\S+)\s+(\S+)\s+(\S+)\s+(\S+)\s+(\S+)\s+([+-]?\d+)([^\t\n]*)", line)
                try:
                    if m is None:
                        raise ValueError
                    tok = m.groups()
                    row = [int(tok[0])] + [float(v) for v in tok[1:8]] + [int(tok[8])]
                    links = [int(v) for v in tok[9].split()]
                except ValueError:
                    continue
                rows.append(row)
                pairs += [(row[0], v) for v in links]
        self.loadMap(rows, instance)
        if pairs:
            arr = np.ascontiguousarray(np.array(pairs, np.int32))
            _lib.check(self.lib.fid_map_add_links(self.h, instance, len(pairs), arr.ctypes.data_as(C.c_void_p)))
        return len(rows)

    @staticmethod
    def _obs(transforms):
        arr = (_lib.fid_transform * max(len(transforms), 1))()
        for i, ft in enumerate(transforms):
            if isinstance(ft, FiducialTransform):
                arr[i].fiducial_id = ft.fiducial_id
                arr[i].translation[:] = ft.transform.translation
                arr[i].rotation[:] = ft.transform.rotation
                arr[i].image_error, arr[i].object_error, arr[i].fiducial_area = ft.image_error, ft.object_error, ft.fiducial_area
            else:
                arr[i].fiducial_id = int(ft["fiducial_id"])
                arr[i].translation[:] = [float(v) for v in ft["translation"]]
                arr[i].rotation[:] = [float(v) for v in ft["rotation"]]
                arr[i].image_error, arr[i].object_error, arr[i].fiducial_area = float(ft["image_error"]), float(ft["object_error"]), float(ft["fiducial_area"])
        return arr

    def transformCallback(self, msg, T_baseCam=None, T_camBase=None, instance=0):
        """msg: FiducialTransformArray or list of transforms.  T_* = 7-vectors (x y z qx qy qz qw) the
        host got from tf (map.cpp:258-273), None when the lookup failed.  Returns fid_robot_pose."""
        transforms = msg.transforms if isinstance(msg, FiducialTransformArray) else list(msg)
        arr = self._obs(transforms)
        bc, cb = _tf(T_baseCam), _tf(T_camBase)
        robot = _lib.fid_robot_pose()
        _lib.check(self.lib.fid_map_update(self.h, instance, len(transforms), C.cast(arr, C.c_void_p), C.byref(bc) if bc is not None else None,
                                           C.byref(cb) if cb is not None else None, C.byref(robot)), "fid_map_update")
        return robot

    def replay(self, messages_per_instance, T_baseCam=None, T_camBase=None):
        """messages_per_instance[i] = list of messages (lists of transforms) for instance i; all
        instances must have the same number of messages.  One kernel launch."""
        ni = self.p.n_instances
        assert len(messages_per_instance) == ni
        n_msgs = len(messages_per_instance[0])
        flat = []
        offsets = np.zeros((ni, n_msgs + 1), np.int32)
        for i, msgs in enumerate(messages_per_instance):
            assert len(msgs) == n_msgs
            for k, m in enumerate(msgs):
                offsets[i, k] = len(flat)
                flat.extend(m)
            offsets[i, n_msgs] = len(flat)
        arr = self._obs(flat)
        robots = (_lib.fid_robot_pose * (ni * n_msgs))()
        bc, cb = _tf(T_baseCam), _tf(T_camBase)
        _lib.check(self.lib.fid_map_update_sequence(self.h, n_msgs, offsets.ctypes.data_as(C.c_void_p), C.cast(arr, C.c_void_p), C.byref(bc) if bc is not None else None,
                                                    C.byref(cb) if cb is not None else None, C.cast(robots, C.c_void_p)), "fid_map_update_sequence")
        return robots

    def update_frames(self, counts, tfs, T_baseCam=None, T_camBase=None, instance=0, asynchronous=False):
        """One message per frame straight from Detector.detect_pose_batch's dense output.  With
        asynchronous=True the fold is only enqueued (it overlaps the next detection); sync() waits."""
        counts = np.ascontiguousarray(counts, np.int32)
        bc, cb = _tf(T_baseCam), _tf(T_camBase)
        if asynchronous:
            _lib.check(self.lib.fid_map_update_frames_async(self.h, instance, len(counts), counts.ctypes.data_as(C.c_void_p), C.cast(tfs, C.c_void_p), MAXM,
                                                            C.byref(bc) if bc is not None else None, C.byref(cb) if cb is not None else None), "fid_map_update_frames_async")
            return None
        robot = _lib.fid_robot_pose()
        _lib.check(self.lib.fid_map_update_frames(self.h, instance, len(counts), counts.ctypes.data_as(C.c_void_p), C.cast(tfs, C.c_void_p), MAXM,
                                                  C.byref(bc) if bc is not None else None, C.byref(cb) if cb is not None else None, C.byref(robot)), "fid_map_update_frames")
        return robot

    def sync(self):
        _lib.check(self.lib.fid_map_sync(self.h))

    TRANSFORM_DTYPE = np.dtype([("fiducial_id", "<i4"), ("reserved", "<i4"), ("translation", "<f8", 3), ("rotation", "<f8", 4), ("image_error", "<f8"),
                                ("object_error", "<f8"), ("fiducial_area", "<f8"), ("rvec", "<f8", 3)])

    def replay_raw(self, offsets: np.ndarray, obs: np.ndarray, T_baseCam=None, T_camBase=None):
        """offsets int32 [n_instances, n_msgs+1] into obs (TRANSFORM_DTYPE records); one launch."""
        offsets = np.ascontiguousarray(offsets, np.int32)
        obs = np.ascontiguousarray(obs)
        assert obs.dtype == self.TRANSFORM_DTYPE and offsets.shape[0] == self.p.n_instances
        bc, cb = _tf(T_baseCam), _tf(T_camBase)
        _lib.check(self.lib.fid_map_update_sequence(self.h, offsets.shape[1] - 1, offsets.ctypes.data_as(C.c_void_p), obs.ctypes.data_as(C.c_void_p),
                                                    C.byref(bc) if bc is not None else None, C.byref(cb) if cb is not None else None, None), "fid_map_update_sequence")

    def entries(self, instance=0):
        cap = self.p.max_fiducials
        arr = (_lib.fid_map_entry * cap)()
        n = C.c_int(0)
        _lib.check(self.lib.fid_map_entries(self.h, instance, cap, C.byref(n), C.cast(arr, C.c_void_p)))
        return [arr[i] for i in range(n.value)]

    def publishMap(self, instance=0) -> FiducialMapEntryArray:  # map.cpp:629-654
        return FiducialMapEntryArray([FiducialMapEntry(e.fiducial_id, e.x, e.y, e.z, e.rx, e.ry, e.rz) for e in self.entries(instance)])

    def clear(self, instance=0):
        _lib.check(self.lib.fid_map_clear(self.h, instance))

    def addFiducial(self, fiducial_id, T_mapBase=None, instance=0):
        """add_fiducial service (addFiducialCallback, map.cpp:821-828): handled by the next transformCallback that observes the id
        (handleAddFiducial, map.cpp:489-535).  T_mapBase = the tf lookup map -> base (7-vector) or None when it fails."""
        mb = _tf(T_mapBase)
        _lib.check(self.lib.fid_map_add_fiducial(self.h, instance, int(fiducial_id), C.byref(mb) if mb is not None else None))

    # ---- published pose (host-side message packing, map.cpp:337-379) ----
    covariance_diagonal = None   # rosparam covariance_diagonal (map.cpp:110-125): six non-zero values or ignored
    publish_6dof_pose = False    # map.cpp:107

    def robotPoseCovariance(self, robot):
        return robot_pose_covariance(robot.variance, self.covariance_diagonal)

    def poseTf(self, robot, T_odomBase=None):
        return pose_tf(robot.t[:], robot.q[:], T_odomBase, self.publish_6dof_pose)

    def refine(self, messages, instance=0, **params):
        """fid_map_refine: batch SE(3) Gauss-Newton over the relative poses the recorded messages contain (new; SURVEY 8f-3).
        messages = list of messages (lists of FiducialTransform-like dicts).  Returns fid_refine_stats."""
        flat, offsets = [], [0]
        for m in messages:
            flat.extend(m)
            offsets.append(len(flat))
        arr = self._obs(flat)
        off = np.ascontiguousarray(np.array(offsets, np.int32))
        p = _lib.fid_refine_params()
        _lib.check(self.lib.fid_map_refine_default_params(C.byref(p)))
        for k, v in params.items():
            if not hasattr(p, k):
                raise AttributeError("unknown refine parameter %r" % k)
            setattr(p, k, v)
        st = _lib.fid_refine_stats()
        _lib.check(self.lib.fid_map_refine(self.h, instance, len(messages), off.ctypes.data_as(C.c_void_p), C.cast(arr, C.c_void_p), C.byref(p), C.byref(st)), "fid_map_refine")
        return st

    def bundle_adjust(self, counts, ids, corners, K, D, fiducial_len=0.14, overrides=None, instance=0, criteria=None):
        """fid_map_bundle_adjust: bundle adjustment of the map from recorded corners (new; DESIGN.md f16).  counts [F], ids [F][m],
        corners [F][m][4][2] as Detector.detect_pose_batch returns them; overrides = {id: length}; criteria = cv2-style (type,
        max_iter, epsilon) or None.  The free entries' poses are updated in place.  Returns (fid_ba_stats, rvecs [F][3],
        tvecs [F][3], status [F], {id: standard deviations of (dtheta, dt)})."""
        counts = np.ascontiguousarray(counts, np.int32)
        ids = np.ascontiguousarray(ids, np.int32)
        F, mm = ids.shape
        corners = np.ascontiguousarray(corners, np.float32).reshape(F, mm, 8)
        ov = dict(overrides or {})
        ov_ids = np.ascontiguousarray(list(ov.keys()), np.int32)
        ov_lens = np.ascontiguousarray(list(ov.values()), np.float64)
        p = _lib.fid_ba_params()
        _lib.check(self.lib.fid_map_ba_default_params(C.byref(p)))
        if criteria is not None:
            p.criteria = _lib.fid_calib_criteria(int(criteria[0]), int(criteria[1]), float(criteria[2]))
        cam = _camera(K, D)
        st = _lib.fid_ba_stats()
        rv, tv, status = np.zeros((F, 3)), np.zeros((F, 3)), np.zeros(F, np.int32)
        ents = self.entries(instance)
        sd = np.zeros((max(len(ents), 1), 6))
        _lib.check(self.lib.fid_map_bundle_adjust(self.h, instance, F, counts.ctypes.data_as(C.c_void_p), ids.ctypes.data_as(C.c_void_p),
                                                  corners.ctypes.data_as(C.c_void_p), mm, C.byref(cam), float(fiducial_len), len(ov_ids),
                                                  ov_ids.ctypes.data_as(C.c_void_p) if len(ov_ids) else None, ov_lens.ctypes.data_as(C.c_void_p) if len(ov_ids) else None,
                                                  C.byref(p), C.byref(st), rv.ctypes.data_as(C.c_void_p), tv.ctypes.data_as(C.c_void_p),
                                                  status.ctypes.data_as(C.c_void_p), sd.ctypes.data_as(C.c_void_p)), "fid_map_bundle_adjust")
        return st, rv, tv, status, {e.fiducial_id: sd[k].copy() for k, e in enumerate(ents)}

    LOCALIZATION_DTYPE = np.dtype(_lib.fid_localization)

    def localize(self, counts, ids, corners, K, D, fiducial_len=0.14, overrides=None, T_camBase=None, instance=0, max_entry_variance=-1):
        """fid_map_localize: per frame, the camera pose that every visible mapped marker's corners determine together, with its
        covariance (new; DESIGN.md f17).  counts [F], ids [F][m], corners [F][m][4][2] as Detector.detect_pose_batch returns them;
        overrides = {id: length}; T_camBase = 7-vector (x y z qx qy qz qw) of the camera mount, or None for the camera's own pose;
        max_entry_variance >= 0 leaves out entries less certain than that.  The map is not changed.  Returns a LOCALIZATION_DTYPE
        array [F] (status 1 pose, 0 no usable mapped marker, -1 no start)."""
        counts = np.ascontiguousarray(counts, np.int32)
        ids = np.ascontiguousarray(ids, np.int32)
        F, mm = ids.shape
        corners = np.ascontiguousarray(corners, np.float32).reshape(F, mm, 8)
        ov = dict(overrides or {})
        ov_ids = np.ascontiguousarray(list(ov.keys()), np.int32)
        ov_lens = np.ascontiguousarray(list(ov.values()), np.float64)
        cam = _camera(K, D)
        cb = _tf(T_camBase)
        out = np.zeros(F, self.LOCALIZATION_DTYPE)
        _lib.check(self.lib.fid_map_localize(self.h, instance, F, counts.ctypes.data_as(C.c_void_p), ids.ctypes.data_as(C.c_void_p), corners.ctypes.data_as(C.c_void_p),
                                             mm, C.byref(cam), float(fiducial_len), len(ov_ids), ov_ids.ctypes.data_as(C.c_void_p) if len(ov_ids) else None,
                                             ov_lens.ctypes.data_as(C.c_void_p) if len(ov_ids) else None, float(max_entry_variance),
                                             C.byref(cb) if cb is not None else None, out.ctypes.data_as(C.POINTER(_lib.fid_localization))), "fid_map_localize")
        return out

    # multi_error_theshold (map.cpp:127-129; its default -1 never switches): the object error below which /fiducial_pose carries
    # the joint pose of localize() instead of the fold's
    multi_error_threshold = -1.0

    def published_pose(self, robot, loc=None):
        """What goes on /fiducial_pose: (t[3], q_xyzw[4], covariance[36]).  The joint pose of a localize() record and its
        covariance when multi_error_threshold >= 0, loc's status is 1 and its object_error is below the threshold; otherwise the
        fold's robot pose with robotPoseCovariance.  covariance_diagonal overrides the diagonal of either (map.cpp:341-345).
        Publication only: the fold and the map are unchanged."""
        if loc is not None and self.multi_error_threshold >= 0 and int(loc["status"]) == 1 and float(loc["object_error"]) < self.multi_error_threshold:
            cov = [float(v) for v in loc["covariance"]]
            d = self.covariance_diagonal
            if d is not None and len(d) == 6 and all(v != 0 for v in d):
                for i in range(6):
                    cov[i * 6 + i] = float(d[i])
            return [float(v) for v in loc["t"]], [float(v) for v in loc["q"]], cov
        return list(robot.t[:]), list(robot.q[:]), self.robotPoseCovariance(robot)

    # multi-GPU merged view (new; SURVEY 8e): local instances are never overwritten by a merge
    def export_table(self, instance=0) -> np.ndarray:
        cap = self.p.max_fiducials
        arr = (_lib.fid_map_record * cap)()
        _lib.check(self.lib.fid_map_export(self.h, instance, C.cast(arr, C.c_void_p)))
        return np.frombuffer(arr, dtype=np.uint8).copy()

    def merge_tables(self, tables: np.ndarray, n_tables: int):
        """Fold n_tables gathered tables (rank order) into the merged view (rebuilt from scratch: idempotent)."""
        tables = np.ascontiguousarray(tables, np.uint8)
        _lib.check(self.lib.fid_map_merge(self.h, n_tables, tables.ctypes.data_as(C.c_void_p)))

    def merged_entries(self):
        cap = self.p.max_fiducials
        arr = (_lib.fid_map_entry * cap)()
        n = C.c_int(0)
        _lib.check(self.lib.fid_map_merged_entries(self.h, cap, C.byref(n), C.cast(arr, C.c_void_p)))
        return [arr[i] for i in range(n.value)]

    def adopt_merged(self, instance=0):
        _lib.check(self.lib.fid_map_adopt_merged(self.h, instance))

    @property
    def table_bytes(self) -> int:
        return self.p.max_fiducials * C.sizeof(_lib.fid_map_record)

    def cuda_stream(self) -> int:
        st = C.c_void_p()
        _lib.check(self.lib.fid_map_stream(self.h, C.byref(st)))
        return st.value or 0

    def export_async(self, device_ptr: int, instance=0):
        _lib.check(self.lib.fid_map_export_async(self.h, instance, C.c_void_p(device_ptr)))

    def merge_device_async(self, device_ptr: int, n_tables: int):
        _lib.check(self.lib.fid_map_merge_device_async(self.h, n_tables, C.c_void_p(device_ptr)))


def robot_pose_covariance(variance, covariance_diagonal=None):
    """Row-major 6x6 covariance of the PoseWithCovarianceStamped on /fiducial_pose: toPose fills the diagonal with the scalar
    variance (transform_with_variance.h:69-84); a covariance_diagonal of six non-zero values overrides it (map.cpp:110-125,341-345)."""
    cov = [0.0] * 36
    diag = [float(variance)] * 6
    if covariance_diagonal is not None and len(covariance_diagonal) == 6 and all(v != 0 for v in covariance_diagonal):
        diag = [float(v) for v in covariance_diagonal]
    for i in range(6):
        cov[i * 6 + i] = diag[i]
    return cov


def pose_tf(t, q, T_odomBase=None, publish_6dof_pose=False):
    """The transform broadcast as map -> odom (or map -> base): outPose = basePose * odom^-1 when the odom lookup succeeded
    (map.cpp:351-365), squashed to x, y, yaw unless publish_6dof_pose (map.cpp:369-379).  Returns (t[3], q_xyzw[4])."""
    t = np.array(t, np.float64)
    R = _q_to_R(q)
    if T_odomBase is not None:
        Ro = _q_to_R(T_odomBase[3:7])
        to = np.array(T_odomBase[:3], np.float64)
        Rinv = Ro.T
        tinv = Rinv @ (-to)
        t = R @ tinv + t
        R = R @ Rinv
    if not publish_6dof_pose:
        t[2] = 0.0
        yaw = _get_rpy(R)[2]
        R = _set_rpy(0.0, 0.0, yaw)
    return t, _R_to_q(R)


# ---- tf2 LinearMath pieces used by the host-side message packing above ------------------------------------
def _q_to_R(q):  # tf2::Matrix3x3::setRotation
    x, y, z, w = [float(v) for v in q]
    d = x * x + y * y + z * z + w * w
    s = 2.0 / d
    xs, ys, zs = x * s, y * s, z * s
    wx, wy, wz, xx, xy, xz, yy, yz, zz = w * xs, w * ys, w * zs, x * xs, x * ys, x * zs, y * ys, y * zs, z * zs
    return np.array([[1.0 - (yy + zz), xy - wz, xz + wy], [xy + wz, 1.0 - (xx + zz), yz - wx], [xz - wy, yz + wx, 1.0 - (xx + yy)]])


def _R_to_q(m):  # tf2::Matrix3x3::getRotation
    tr = m[0][0] + m[1][1] + m[2][2]
    q = [0.0] * 4
    if tr > 0.0:
        s = math.sqrt(tr + 1.0)
        q[3] = s * 0.5
        s = 0.5 / s
        q[0], q[1], q[2] = (m[2][1] - m[1][2]) * s, (m[0][2] - m[2][0]) * s, (m[1][0] - m[0][1]) * s
    else:
        i = (2 if m[1][1] < m[2][2] else 1) if m[0][0] < m[1][1] else (2 if m[0][0] < m[2][2] else 0)
        j, k = (i + 1) % 3, (i + 2) % 3
        s = math.sqrt(m[i][i] - m[j][j] - m[k][k] + 1.0)
        q[i] = s * 0.5
        s = 0.5 / s
        q[3] = (m[k][j] - m[j][k]) * s
        q[j] = (m[j][i] + m[i][j]) * s
        q[k] = (m[k][i] + m[i][k]) * s
    return np.array(q)


def _get_rpy(m):  # tf2::Matrix3x3::getRPY
    if abs(m[2][0]) >= 1.0:
        delta = math.atan2(m[2][1], m[2][2])
        return (delta, math.pi / 2.0, 0.0) if m[2][0] < 0 else (delta, -math.pi / 2.0, 0.0)
    pitch = -math.asin(m[2][0])
    c = math.cos(pitch)
    return math.atan2(m[2][1] / c, m[2][2] / c), pitch, math.atan2(m[1][0] / c, m[0][0] / c)


def _set_rpy(roll, pitch, yaw):  # tf2::Matrix3x3::setRPY
    ci, cj, ch = math.cos(roll), math.cos(pitch), math.cos(yaw)
    si, sj, sh = math.sin(roll), math.sin(pitch), math.sin(yaw)
    cc, cs, sc, ss = ci * ch, ci * sh, si * ch, si * sh
    return np.array([[cj * ch, sj * sc - cs, sj * cc + ss], [cj * sh, sj * ss + cc, sj * cs - sc], [-sj, cj * si, cj * ci]])


class JpegDecoder:
    """fid_jpeg_*: the cv::imdecode that compressed_image_transport runs in front of imageCallback (aruco_detect.cpp:332,348;
    launch default transport `compressed`), with the Huffman stage on host threads and everything after it on the device.
    decode(list of bytes-like JPEG streams, device pointer) writes BGR8 frames into device memory
    (FiducialsNode.detector_device_alloc / fid_device_alloc) for submit_batch(..., on_device=True)."""

    def __init__(self, max_width, max_height, max_batch, device=0, n_threads=0):
        self.lib = _lib.load()
        h = C.c_void_p()
        _lib.check(self.lib.fid_jpeg_create(device, max_width, max_height, max_batch, n_threads, C.byref(h)), "fid_jpeg_create")
        self.h = h

    def decode(self, streams, device_ptr, width, height, row_stride=None, frame_stride=None, sync=True):
        n = len(streams)
        bufs = [np.frombuffer(bytes(s) if not isinstance(s, np.ndarray) else s, np.uint8) for s in streams]
        ptrs = (C.c_void_p * n)(*[b.ctypes.data for b in bufs])
        sizes = (C.c_size_t * n)(*[b.size for b in bufs])
        status = np.zeros(n, np.int32)
        rs = row_stride or width * 3
        fs = frame_stride or rs * height
        _lib.check(self.lib.fid_jpeg_decode_batch(self.h, n, ptrs, sizes, width, height, C.c_void_p(int(device_ptr)), rs, fs, status.ctypes.data_as(C.c_void_p)), "fid_jpeg_decode_batch")
        self._keep = bufs
        if sync:
            self.sync()
        return status

    def sync(self):
        _lib.check(self.lib.fid_jpeg_sync(self.h))

    def stats(self):
        a, b, c = C.c_double(0), C.c_double(0), C.c_double(0)
        _lib.check(self.lib.fid_jpeg_last_stats(self.h, C.byref(a), C.byref(b), C.byref(c)))
        return {"host_decode_ms": a.value, "h2d_bytes": b.value, "device_ms": c.value}

    def close(self):
        if self.h:
            self.lib.fid_jpeg_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
