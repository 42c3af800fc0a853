"""Detection and the board stages on dense calibration targets (tests/dense_cases.py) against cv2, up to and past the per-frame
capacities: 4096 raw quad candidates, 512 selected candidates and 256 markers.  The cases cross the sizes at which k_sort_group keeps
its close-pair matrix (615 raw candidates) and its sorted quads (1537) in global memory and stages more matrix words per lane
(2049), at which k_finish's loops and the board stages run a second and third stride, and at which the capacity status is returned.
Tolerances as in tests/test_gpu_parity.py: candidates bit-exact, ids and order identical, corners within 1e-3 px, poses within 1e-3."""
import ctypes as C
import functools

import cv2
import numpy as np
import pytest

import dense_cases as dc
from fiducials_b200 import _lib, synth
from fiducials_b200.board import charuco_board, grid_board
from fiducials_b200.node import MAXM, Detector, _camera, default_params
from oracle import aruco_oracle as ao
import board_oracle as bo
import charuco_oracle as co

pytestmark = pytest.mark.gpu

FID_OK, FID_ERR_CAPACITY = 0, -5
FLEN = 0.14
# one case per band of the raw-candidate count: <= 614, 615..1536, 1537..2048, 2049..3072, 3073..4096
BAND_CASES = ["grid_6x4", "grid_10x6", "grid_14x8", "grid_16x9", "grid_20x12"]


@pytest.fixture(params=["simt", "mma"])
def thresh(request, monkeypatch):
    """Both threshold kernels (FID_THRESH is read by fid_create)."""
    if request.param == "mma":
        monkeypatch.setenv("FID_THRESH", "mma")
    else:
        monkeypatch.delenv("FID_THRESH", raising=False)
    return request.param


def _detector(name, max_batch=1, **overrides):
    c = dc.CASES[name]
    return Detector(default_params(dictionary=c["dict_id"], **dict(c["params"], **overrides)), 0, c["W"], c["H"], max_batch)


@functools.lru_cache(maxsize=None)
def _frame(name):
    return dc.render(name)


@functools.lru_cache(maxsize=None)
def _oracle(name, **overrides):
    """cv2's ids, corners and per-marker poses of a case."""
    c = dc.CASES[name]
    K, D = dc.camera(name)
    kw = dict(c["params"], **overrides)
    if c["inverted"]:
        kw["detectInvertedMarker"] = True
    return ao.detect_and_pose(_frame(name)[0], c["dict_id"], K, D, FLEN, **kw)


def _assert_markers(ids, corners, rids, rcorners, what=""):
    assert np.asarray(ids).tolist() == np.asarray(rids).tolist(), what
    if len(rids):
        assert np.abs(np.asarray(corners).reshape(-1, 4, 2) - rcorners).max() <= 1e-3, what


def _assert_poses(tfs, first, fields, what=""):
    for m, f in enumerate(fields):
        t = tfs[first + m]
        assert t.fiducial_id == f["fiducial_id"], (what, m)
        assert np.abs(np.array(t.translation[:]) - f["translation"]).max() <= 1e-3, (what, m)
        assert np.abs(np.array(t.rotation[:]) - f["rotation"]).max() <= 1e-3, (what, m)


def _raw_detect(det, bgr, max_markers=MAXM):
    """fid_detect through ctypes (the wrapper raises on a nonzero status): (status, n, ids, corners [n, 4, 2])."""
    H, W = bgr.shape[:2]
    ids = np.full(max_markers, -7, np.int32)
    corners = np.zeros((max_markers, 8), np.float32)
    n = C.c_int(-1)
    st = det.lib.fid_detect(det.h, bgr.ctypes.data_as(C.c_void_p), W, H, W * 3, max_markers, C.byref(n), ids.ctypes.data_as(C.c_void_p),
                            corners.ctypes.data_as(C.c_void_p))
    return st, n.value, ids[: max(n.value, 0)].copy(), corners[: max(n.value, 0)].reshape(-1, 4, 2).copy()


def _batch_out(nf, pose):
    return (np.full(nf, -7, np.int32), np.full((nf, MAXM), -7, np.int32), np.zeros((nf, MAXM, 8), np.float32),
            (_lib.fid_transform * (nf * MAXM))() if pose else None)


def _raw_batch(det, frames, K=None, D=None):
    """fid_detect_pose_batch through ctypes: (status, counts, ids, corners [nf, MAXM, 4, 2], transforms)."""
    frames = np.ascontiguousarray(frames)
    nf, H, W = frames.shape[:3]
    cam = _camera(K, D) if K is not None else None
    counts, ids, corners, tfs = _batch_out(nf, cam is not None)
    st = det.lib.fid_detect_pose_batch(det.h, nf, frames.ctypes.data_as(C.c_void_p), 0, W, H, W * 3, W * 3 * H, C.byref(cam) if cam is not None else None,
                                       FLEN, 0, None, None, MAXM, counts.ctypes.data_as(C.c_void_p), ids.ctypes.data_as(C.c_void_p),
                                       corners.ctypes.data_as(C.c_void_p), C.cast(tfs, C.c_void_p) if tfs is not None else None)
    return st, counts, ids, corners.reshape(nf, MAXM, 4, 2), tfs


def _raw_submit_collect(det, frames):
    """fid_submit_batch + fid_collect_batch through ctypes, no camera: (submit status, collect status, counts, ids, corners)."""
    frames = np.ascontiguousarray(frames)
    nf, H, W = frames.shape[:3]
    s1 = det.lib.fid_submit_batch(det.h, nf, frames.ctypes.data_as(C.c_void_p), 0, W, H, W * 3, W * 3 * H, None, FLEN, 0, None, None)
    counts, ids, corners, _ = _batch_out(nf, False)
    s2 = det.lib.fid_collect_batch(det.h, MAXM, counts.ctypes.data_as(C.c_void_p), ids.ctypes.data_as(C.c_void_p), corners.ctypes.data_as(C.c_void_p), None)
    return s1, s2, counts, ids, corners.reshape(nf, MAXM, 4, 2)


def _assert_candidates(det, name):
    quads, scale, clen = det.debug_candidates()
    ref = ao.quad_candidates(ao.gray(_frame(name)[0]), dc.oracle_params(name))
    assert len(quads) == len(ref), (name, len(quads), len(ref))
    assert np.array_equal(scale, [s for s, _, _ in ref]) and np.array_equal(clen, [n for _, _, n in ref]), name
    assert np.array_equal(quads, np.array([q for _, q, _ in ref]).reshape(-1, 4, 2)), name


# ---- 2. parity across the size switches -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", BAND_CASES)
def test_dense_board_matches_cv2(thresh, name):
    """Raw candidates bit-exact (quads, scale, contour length), markers identical to cv2's, poses of the batch call within 1e-3."""
    bgr, _ = _frame(name)
    K, D = dc.camera(name)
    rids, rcorners, _, _, fields = _oracle(name)
    assert len(rids) == dc.MARKERS[name]
    det = _detector(name)
    try:
        ids, corners = det.detect(bgr)
        _assert_candidates(det, name)
        _assert_markers(ids, corners, rids, rcorners, name)
        counts, bids, bcorners, tfs = det.detect_pose_batch(bgr[None], K, D, FLEN)
        n = int(counts[0])
        _assert_markers(bids[0, :n], bcorners[0, :n], rids, rcorners, name)
        _assert_poses(tfs, 0, fields, name)
    finally:
        det.close()


@pytest.mark.parametrize("name", ["grid_10x6", "grid_20x12"])
def test_dense_board_contour_refinement(thresh, name):
    """CORNER_REFINE_CONTOUR launches k_contour_refine over max_sel candidate slots per frame.  Tolerance of
    tests/test_gpu_parity.py::test_corner_refine_contour: these markers have sides of 100 contour points and more, where OpenCV forms
    the normal equations through the BLAS sgemm of its build."""
    bgr, _ = _frame(name)
    rids, rcorners, _, _, _ = _oracle(name, cornerRefinementMethod=cv2.aruco.CORNER_REFINE_CONTOUR)
    assert len(rids) == dc.MARKERS[name]
    det = _detector(name, cornerRefinementMethod=2)
    try:
        ids, corners = det.detect(bgr)
    finally:
        det.close()
    assert ids.tolist() == rids.tolist()
    assert np.abs(corners - rcorners).max() <= 2e-2


def test_dense_inverted_board(thresh):
    """detectInvertedMarker (k_sort_group<true>) on a white-on-black board of 2 096 raw candidates."""
    name = "grid_14x8_inverted"
    bgr, _ = _frame(name)
    K, D = dc.camera(name)
    rids, rcorners, _, _, fields = _oracle(name)
    assert len(rids) == dc.MARKERS[name]
    det = _detector(name)
    try:
        det.set_detect_inverted_marker(True)
        ids, corners = det.detect(bgr)
        _assert_candidates(det, name)
        _assert_markers(ids, corners, rids, rcorners, name)
        counts, bids, bcorners, tfs = det.detect_pose_batch(bgr[None], K, D, FLEN)
        _assert_markers(bids[0, : counts[0]], bcorners[0, : counts[0]], rids, rcorners, name)
        _assert_poses(tfs, 0, fields, name)
    finally:
        det.close()


# ---- 3. batch isolation -------------------------------------------------------------------------------------------------------------
def _mixed_chunk(dense):
    """One chunk: a dense frame, a C2 frame (DICT_6X6_250 markers, candidates without a DICT_5X5_1000 marker), a blank frame and a
    second dense frame (1920 x 1080)."""
    c2 = synth.make_config_frame("C2", 3)[0]
    blank = np.full_like(c2, 128)
    return np.ascontiguousarray(np.stack([_frame(dense)[0], c2, blank, _frame("grid_14x8")[0]]))


@pytest.mark.parametrize("dense", ["grid_20x12", "grid_24x14"])
def test_batch_frames_stay_apart(thresh, dense):
    """Every frame of a chunk gives its own single-frame result and cv2's, next to a frame at 3 576 raw candidates and next to one past
    the per-frame raw capacity (4 696): a frame that wrote into its neighbour's [max_raw] slice would show here."""
    frames = _mixed_chunk(dense)
    over = dc.CASES[dense]["band"] == "gt4096"
    K, D = dc.camera("grid_14x8")
    det = _detector("grid_14x8", max_batch=4)
    try:
        st, counts, ids, corners, tfs = _raw_batch(det, frames, K, D)
        assert st == (FID_ERR_CAPACITY if over else FID_OK)
        for f in range(len(frames)):
            n = int(counts[f])
            if over and f == 0:  # the frame past the capacity: some of its markers, each one rendered
                assert 0 < n <= MAXM and set(ids[0, :n].tolist()) <= _frame(dense)[1]
                continue
            rids, rcorners, _, _, fields = ao.detect_and_pose(frames[f], 7, K, D, FLEN)
            _assert_markers(ids[f, :n], corners[f, :n], rids, rcorners, "frame %d" % f)
            _assert_poses(tfs, f * MAXM, fields, "frame %d" % f)
            sids, scorners = det.detect(frames[f])
            assert np.array_equal(sids, ids[f, :n]) and np.array_equal(scorners, corners[f, :n]), f
    finally:
        det.close()


# ---- 4. capacity contract -----------------------------------------------------------------------------------------------------------
def test_exactly_256_markers():
    name = "grid_16x16"
    bgr, _ = _frame(name)
    rids, rcorners, _, _, _ = _oracle(name)
    assert len(rids) == MAXM
    det = _detector(name)
    try:
        st, n, ids, corners = _raw_detect(det, bgr)
        assert st == FID_OK and n == MAXM
        _assert_markers(ids, corners, rids, rcorners)
        st, counts, bids, bcorners, _ = _raw_batch(det, bgr[None])
        assert st == FID_OK and counts[0] == MAXM
        _assert_markers(bids[0], bcorners[0], rids, rcorners)
    finally:
        det.close()


@pytest.mark.parametrize("name", ["grid_22x13", "grid_28x16_few"])
def test_more_than_256_markers(name):
    """Under 4 096 raw and at most 512 selected candidates but more than 256 markers: FID_ERR_CAPACITY and cv2's first 256 markers, in
    order, with cv2's corners, from fid_detect and from the batch calls."""
    bgr, _ = _frame(name)
    rids, rcorners, _, _, _ = _oracle(name)
    assert len(rids) == dc.MARKERS[name] > MAXM
    det = _detector(name, max_batch=2)
    try:
        st, n, ids, corners = _raw_detect(det, bgr)
        assert st == FID_ERR_CAPACITY and n == MAXM
        _assert_markers(ids, corners, rids[:MAXM], rcorners[:MAXM], name)
        frames = np.ascontiguousarray(np.stack([bgr, bgr[::-1, ::-1]]))  # and the board turned by half a turn
        rids2, rcorners2 = ao.detect(frames[1], dc.CASES[name]["dict_id"], **dc.CASES[name]["params"])
        assert len(rids2) > MAXM
        st, counts, bids, bcorners, _ = _raw_batch(det, frames)
        assert st == FID_ERR_CAPACITY and counts.tolist() == [MAXM, MAXM]
        _assert_markers(bids[0], bcorners[0], rids[:MAXM], rcorners[:MAXM], name)
        _assert_markers(bids[1, : counts[1]], bcorners[1, : counts[1]], rids2[:MAXM], rcorners2[:MAXM], name + " mirrored")
        s1, s2, counts, cids, ccorners = _raw_submit_collect(det, frames)
        assert s1 == FID_OK and s2 == FID_ERR_CAPACITY and np.array_equal(cids, bids) and np.array_equal(ccorners, bcorners)
    finally:
        det.close()


def test_more_than_512_selected():
    name = "grid_32x18_few"
    bgr, rendered = _frame(name)
    det = _detector(name)
    try:
        st, n, ids, _ = _raw_detect(det, bgr)
        assert st == FID_ERR_CAPACITY and 0 < n <= MAXM and set(ids.tolist()) <= rendered
        st, counts, bids, _, _ = _raw_batch(det, bgr[None])
        assert st == FID_ERR_CAPACITY and counts[0] == n and np.array_equal(bids[0, :n], ids)
        assert det.last_counters()["selected"] == 512  # the selected list stops at the per-frame capacity
    finally:
        det.close()


@pytest.mark.parametrize("name", ["grid_24x14", "grid_18x14_4k"])
def test_more_than_4096_raw_candidates(name):
    """Past the raw-candidate capacity the kept candidates are the ones that won the slot race of k_approx: no particular subset can be
    asserted, only the status and that every marker returned was rendered.  grid_18x14_4k has 252 markers (under the marker capacity)
    and 4 200 raw candidates."""
    bgr, rendered = _frame(name)
    det = _detector(name, max_batch=2)
    try:
        st, n, ids, _ = _raw_detect(det, bgr)
        assert st == FID_ERR_CAPACITY and 0 < n <= MAXM and set(ids.tolist()) <= rendered
        frames = np.ascontiguousarray(np.stack([bgr, bgr]))
        st, counts, bids, _, _ = _raw_batch(det, frames, *dc.camera(name))
        assert st == FID_ERR_CAPACITY
        s1, s2, ccounts, cids, _ = _raw_submit_collect(det, frames)
        assert s1 == FID_OK and s2 == FID_ERR_CAPACITY
        for f in range(2):
            for cn, ci in ((counts[f], bids[f]), (ccounts[f], cids[f])):
                assert 0 < cn <= MAXM and set(ci[:cn].tolist()) <= rendered
    finally:
        det.close()


def test_multi_dictionary_total_past_256():
    """fid_detect_multi_dict with the same dictionary listed twice on 144 markers: 288 in all, FID_ERR_CAPACITY with the first 256 of
    the concatenation written."""
    name = "grid_16x9"
    bgr, _ = _frame(name)
    rids, rcorners, _, _, _ = _oracle(name)
    det = _detector(name)
    try:
        det.set_dictionaries([7, 7])
        ids = np.full(MAXM, -7, np.int32)
        corners = np.zeros((MAXM, 8), np.float32)
        di = np.full(MAXM, -7, np.int32)
        n = C.c_int(-1)
        H, W = bgr.shape[:2]
        st = det.lib.fid_detect_multi_dict(det.h, bgr.ctypes.data_as(C.c_void_p), W, H, W * 3, MAXM, C.byref(n), ids.ctypes.data_as(C.c_void_p),
                                           corners.ctypes.data_as(C.c_void_p), di.ctypes.data_as(C.c_void_p))
        assert st == FID_ERR_CAPACITY and n.value == MAXM
        k = len(rids)
        _assert_markers(ids, corners, np.concatenate([rids, rids])[:MAXM], np.concatenate([rcorners, rcorners])[:MAXM])
        assert di.tolist() == [0] * k + [1] * (MAXM - k)
    finally:
        det.close()


# ---- 5. board stages at full size ---------------------------------------------------------------------------------------------------
def test_board_pose_960_points():
    """k_board_pose over a GridBoard of 240 detected markers (960 points staged in shared memory), against Board.matchImagePoints +
    solvePnP on the device's own detections, with the board oracle's tolerance."""
    name = "grid_20x12"
    bgr, _ = _frame(name)
    K, D = dc.camera(name)
    board = grid_board((20, 12), 0.04, 0.01)
    det = _detector(name)
    try:
        det.set_boards([board])
        counts, ids, corners, _ = det.detect_pose_batch(bgr[None], K, D, FLEN)
        n = int(counts[0])
        assert n == 240
        got = bo.record_dict(det.last_board_poses()[0][0])
        ref = bo.board_pose(board, ids[0, :n], corners[0, :n], K, D)
        assert ref["n_points"] == 960
        bo.assert_matches(got, ref, name)
    finally:
        det.close()


def test_charuco_187_corners():
    """k_charuco on an 18 x 12 ChArUco board: 108 markers and 187 chessboard corners, more than one 128-wide stride of each."""
    name = "charuco_18x12"
    bgr, _ = _frame(name)
    K, D = dc.camera(name)
    board = charuco_board((18, 12), 0.04, 0.03)
    assert board.n_corners == 187
    det = _detector(name)
    try:
        det.set_charuco_boards([board])
        counts, ids, corners, _ = det.detect_pose_batch(bgr[None], K, D, FLEN)
        n = int(counts[0])
        assert n == 108
        rec, cid, cxy = det.last_charuco()[0][0]
        cvb = co.cv_board((18, 12), 0.04, 0.03)
        ri, rx, rp = co.full(cvb, bgr, ids[0, :n], corners[0, :n].reshape(-1, 8), K, D)
        assert len(ri) > 128
        if rp["status"] == 1 and len(ri) == len(cid) and not np.array_equal(rx, cxy):
            rp = co.pose(cvb, cid, cxy, K, D)  # cv2's pose on the device's corners: a corner that moved moves the pose too
        got = dict(status=int(rec.status), rvec=np.array(rec.rvec[:]), tvec=np.array(rec.tvec[:]), rotation=np.array(rec.rotation[:]),
                   image_error=float(rec.image_error))
        co.assert_matches(cid, cxy, got, ri, rx, rp, name)
        assert got["status"] == 1
    finally:
        det.close()
