"""Recovery of missed board markers on the device (fid_set_marker_refinement, fid_refine_detected_markers) against the host build of
the same arithmetic and against cv2.aruco.ArucoDetector.refineDetectedMarkers, on cv2's own detected and rejected lists."""
import ctypes as C

import cv2
import numpy as np
import pytest

from fiducials_b200 import _lib
from fiducials_b200.board import charuco_board, grid_board
from fiducials_b200.node import MAXM, Detector, default_params
import marker_refine_oracle as mo
from test_hostsim_marker_refine import D_REF, D_ZERO, H, K_SYN, W, charuco_scene, grid_scene, hs_refine, lists

pytestmark = pytest.mark.gpu

FID_MAX_BOARDS = 16  # include/fiducials_b200.h

_worst = {"host": 0.0, "cv2": 0.0, "recovered": 0}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\ndevice refinement: %d markers recovered, max |d corner| vs host %.3g px, vs cv2 %.3g px" % (_worst["recovered"], _worst["host"], _worst["cv2"]))


def _detector(method=cv2.aruco.CORNER_REFINE_SUBPIX, rel_win=100.0, refine=(10.0, 3.0, True)):
    det = Detector(default_params(dictionary=mo.DICT, cornerRefinementMethod=method, relativeCornerRefinmentWinSize=rel_win), max_width=W, max_height=H)
    det.set_marker_refinement(*refine)
    return det


def check(det, gray, grids, charucos, ids, corners, rej, K=None, D=None, refine=(10.0, 3.0, True), method=cv2.aruco.CORNER_REFINE_SUBPIX, rel_win=100.0,
          what=""):
    """The device against the host build (identical recoveries, corners within 1e-4 px) and against cv2 (identical recoveries, corners
    bit-identical without cornerSubPix, within 1e-3 px with it)."""
    det.set_boards(grids)
    det.set_charuco_boards(charucos)
    boards = list(grids) + list(charucos)
    labels = list(range(len(grids))) + [FID_MAX_BOARDS + c for c in range(len(charucos))]
    di, dc, dr, dx, db = det.refine_markers(cv2.cvtColor(gray, cv2.COLOR_GRAY2BGR), ids, corners, rej, K, D)
    hi, hc, hr, hx, hb, _ = hs_refine(gray, boards, ids, corners, rej, K, D, refine, method, rel_win)
    assert di.tolist() == hi.tolist() and dx.tolist() == hx and db.tolist() == [labels[b] for b in hb], (what, di, hi, dx, hx)
    assert np.array_equal(dr, hr), what
    dh = float(np.abs(dc - hc).max()) if len(dc) else 0.0
    assert dh <= 1e-4, (what, dh)
    ri, rc, rr, rx, rb, _ = mo.refine(mo.detector(refine, cornerRefinementMethod=method, relativeCornerRefinmentWinSize=rel_win), gray, boards, ids,
                                      corners, rej, K, D)
    assert di.tolist() == ri.tolist() and dx.tolist() == rx, (what, di, ri)
    assert np.array_equal(dr, rr), what
    n0 = len(ids)
    d2 = float(np.abs(dc[n0:] - rc[n0:]).max()) if len(dc) > n0 else 0.0
    assert d2 <= (1e-3 if method == cv2.aruco.CORNER_REFINE_SUBPIX else 0.0), (what, d2)
    _worst["host"] = max(_worst["host"], dh)
    _worst["cv2"] = max(_worst["cv2"], d2)
    _worst["recovered"] += len(dx)
    return dx


@pytest.mark.parametrize("camera", ["none", "D_zero", "D_ref"])
def test_grid_boards(camera):
    rng = np.random.default_rng(60)
    K, D = (None, None) if camera == "none" else (K_SYN, D_ZERO if camera == "D_zero" else D_REF)
    det = _detector()
    for k in range(6):
        size = (int(rng.integers(2, 11)), int(rng.integers(2, 11)))
        board, g = grid_scene(rng, size, ["near", "far", "oblique"][k % 3], n_damaged=int(rng.integers(1, 5)))
        ids, corners, rej = lists(g)
        check(det, g, [board], [], ids, corners, rej, K, D, what="grid %d %s" % (k, size))


@pytest.mark.parametrize("refine", [(10.0, 3.0, False), (10.0, -1.0, True), (3.0, 3.0, True), (40.0, 3.0, True)])
@pytest.mark.parametrize("method", [cv2.aruco.CORNER_REFINE_NONE, cv2.aruco.CORNER_REFINE_SUBPIX])
def test_parameters(refine, method):
    rng = np.random.default_rng(61)
    det = _detector(method, 0.3, refine)
    for k in range(3):
        board, g = grid_scene(rng, (6, 5), ["near", "oblique"][k % 2], n_damaged=4)
        ids, corners, rej = lists(g, method)
        for K in (None, K_SYN):
            check(det, g, [board], [], ids, corners, rej, K, D_ZERO, refine, method, 0.3, what="%s %d" % (refine, k))


def test_marker_and_charuco_boards():
    """A grid board and a ChArUco board set together: the grid is refined first, the ChArUco board on what it left."""
    rng = np.random.default_rng(62)
    det = _detector()
    total = 0
    for k in range(4):
        ch, g = charuco_scene(rng, (5, 4), "near", n_damaged=3)
        ids, corners, rej = lists(g)
        grid = grid_board((3, 3), 0.04, 0.01, ids=np.arange(200, 209))  # not in the frame: nothing to recover
        for K in (None, K_SYN):
            total += len(check(det, g, [grid], [ch], ids, corners, rej, K, D_ZERO, what="charuco %d" % k))
            total += len(check(det, g, [], [ch, ch], ids, corners, rej, K, D_ZERO, what="charuco twice %d" % k))
    assert total > 0


def test_edge_cases_and_errors():
    rng = np.random.default_rng(63)
    board, g = grid_scene(rng, (5, 4), "near", n_damaged=3, kinds=("stripe",))
    ids, corners, rej = lists(g)
    det = _detector()
    for K in (None, K_SYN):
        assert check(det, g, [board], [], ids[:0], corners[:0], rej, K, D_ZERO, what="no detections").tolist() == []
        assert check(det, g, [board], [], ids, corners, rej[:0], K, D_ZERO, what="no rejected").tolist() == []
        check(det, g, [board], [], np.concatenate([ids, ids[:1]]), np.concatenate([corners, corners[:1] + 0.3]), rej, K, D_ZERO, what="repeated")
    bgr = cv2.cvtColor(g, cv2.COLOR_GRAY2BGR)
    # the option off, no board, bad parameters
    off = Detector(default_params(dictionary=mo.DICT), max_width=W, max_height=H)
    off.set_boards([board])
    with pytest.raises(_lib.FidError):
        off.refine_markers(bgr, ids, corners, rej)
    with pytest.raises(_lib.FidError):
        off.set_marker_refinement(min_rep_distance=0.0)
    with pytest.raises(_lib.FidError):
        off.set_marker_refinement(min_rep_distance=float("nan"))
    none = _detector()
    with pytest.raises(_lib.FidError):
        none.refine_markers(bgr, ids, corners, rej)
    # turned off again
    det.set_boards([board])
    det.set_marker_refinement(None)
    with pytest.raises(_lib.FidError):
        det.refine_markers(bgr, ids, corners, rej)
    det.set_marker_refinement()
    # capacity: no room for the recovered markers, nothing written
    n = len(ids)
    oi = np.zeros(n, np.int32)
    oi[:] = ids
    oc = np.ascontiguousarray(corners.reshape(-1, 8)).copy()
    rj = np.ascontiguousarray(rej.reshape(-1, 8))
    ri, rb, nout = np.zeros(MAXM, np.int32), np.zeros(MAXM, np.int32), C.c_int(-1)
    st = det.lib.fid_refine_detected_markers(det.h, bgr.ctypes.data_as(C.c_void_p), W, H, bgr.strides[0], n, oi.ctypes.data_as(C.c_void_p),
                                             oc.ctypes.data_as(C.c_void_p), n, len(rj), rj.ctypes.data_as(C.c_void_p), None, C.byref(nout),
                                             ri.ctypes.data_as(C.c_void_p), rb.ctypes.data_as(C.c_void_p))
    assert st == -5 and nout.value == -1 and np.array_equal(oi, ids)
    # out-of-range sizes
    for bad_n, bad_rej in ((-1, len(rj)), (n, -1), (n, _lib.FID_MAX_REJECTED + 1)):
        st = det.lib.fid_refine_detected_markers(det.h, bgr.ctypes.data_as(C.c_void_p), W, H, bgr.strides[0], bad_n, oi.ctypes.data_as(C.c_void_p),
                                                 oc.ctypes.data_as(C.c_void_p), n, bad_rej, rj.ctypes.data_as(C.c_void_p), None, C.byref(nout),
                                                 ri.ctypes.data_as(C.c_void_p), rb.ctypes.data_as(C.c_void_p))
        assert st == -1


def test_batch_outputs_unchanged():
    """With refinement set, the batch calls launch the same kernels and return the same bytes as a handle that never set it."""
    rng = np.random.default_rng(64)
    frames = []
    for k in range(3):
        board, g = grid_scene(rng, (5, 4), "near", n_damaged=2)
        frames.append(cv2.cvtColor(g, cv2.COLOR_GRAY2BGR))
    frames = np.ascontiguousarray(np.stack(frames))
    outs = []
    for on in (False, True):
        det = Detector(default_params(dictionary=mo.DICT), max_width=W, max_height=H, max_batch=4)
        det.set_boards([board])
        if on:
            det.set_marker_refinement()
        counts, ids, corners, tfs = det.detect_pose_batch(frames, K_SYN, D_ZERO, 0.04)
        c = (C.c_int64 * 8)()
        nc = C.c_int(0)
        _lib.check(det.lib.fid_last_counters(det.h, c, 8, C.byref(nc)))
        outs.append((counts.copy(), ids.copy(), corners.copy(), bytes(tfs), c[6]))
    assert all(np.array_equal(a, b) for a, b in zip(outs[0][:3], outs[1][:3])) and outs[0][3] == outs[1][3] and outs[0][4] == outs[1][4]
