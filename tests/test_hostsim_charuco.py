"""ChArUco corners and pose (fiducials_b200/csrc/charuco.cuh, compiled for the host from tests/hostsim/charuco_hostsim.cpp) against
cv2.aruco.CharucoDetector.detectBoard with given markers + CharucoBoard.matchImagePoints + cv2.solvePnP, and the layout of
fiducials_b200.board.charuco_board against cv2.aruco.CharucoBoard.  CPU only."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import cv2
import numpy as np
import pytest

from fiducials_b200 import synth
from fiducials_b200.board import charuco_board
import charuco_oracle as co

_HERE = os.path.dirname(os.path.abspath(__file__))
_harness = None


def _load():
    """g++ build of the harness into a temporary directory (the tree may be read-only), once per session, without FMA contraction
    like the device build."""
    global _harness
    if _harness is None:
        tmp = tempfile.mkdtemp(prefix="fid_charuco_hostsim_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "libfid_charuco_hostsim.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, os.path.join(_HERE, "hostsim", "charuco_hostsim.cpp")])
        _harness = C.CDLL(so)
    return _harness


_vp = C.c_void_p


def _p(a):
    return None if a is None else a.ctypes.data_as(_vp)


def hs_detect(board, gray, ids, corners, K=None, D=None):
    """charuco.cuh on the host: (corner ids, corners, pose dict) for a fiducials_b200.board.CharucoBoard."""
    gray = np.ascontiguousarray(gray, np.uint8)
    H, W = gray.shape
    nc = board.n_corners
    oi, ox, rec = np.zeros(nc + 1, np.int32), np.zeros((nc + 1, 2), np.float32), np.zeros(16)
    ids = np.ascontiguousarray(ids, np.int32).reshape(-1)
    corners = np.ascontiguousarray(corners, np.float32).reshape(-1, 8)
    Ka = None if K is None else np.ascontiguousarray(K, np.float64).reshape(9)
    Da = None if K is None else np.ascontiguousarray(D, np.float64).reshape(-1)[:5]
    bids = np.ascontiguousarray(board.ids, np.int32)
    n = _load().hs_charuco_detect(board.size[0], board.size[1], C.c_float(board.square_length), C.c_float(board.marker_length), int(board.legacy), _p(bids),
                                  board.min_markers, int(board.check_markers), _p(gray), W, H, len(ids), _p(ids), _p(corners), _p(Ka), _p(Da), co.REFINE_WIN,
                                  co.REFINE_MAX_ITER, C.c_double(co.REFINE_MIN_ACC), _p(oi), _p(ox), _p(rec))
    assert n >= 0
    pose = dict(status=int(rec[1]), rvec=rec[2:5].copy(), tvec=rec[5:8].copy(), rotation=rec[8:12].copy(), image_error=float(rec[12]))
    return oi[:n].copy(), ox[:n].copy(), pose


def cv_of(board):
    return co.cv_board(board.size, board.square_length, board.marker_length, board.ids, board.legacy)


_worst = {"corner": 0.0, "pose": 0.0, "corners": 0, "identical": 0}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nChArUco vs cv2: %d of %d corners bit-identical, max |d corner| = %.3g px, max |d rvec|,|d tvec| = %.3g"
          % (_worst["identical"], _worst["corners"], _worst["corner"], _worst["pose"]))


def check(board, gray, ids, corners, K=None, D=None, what=""):
    gi, gx, gp = hs_detect(board, gray, ids, corners, K, D)
    cvb = cv_of(board)
    ri, rx, rp = co.full(cvb, cv2.cvtColor(gray, cv2.COLOR_GRAY2BGR), ids, corners, K, D, board.min_markers, board.check_markers)
    if rp["status"] == 1 and len(ri) == len(gi) and not np.array_equal(rx, gx):
        rp = co.pose(cvb, gi, gx, K, D)  # the pose of cv2 on the same corners: a corner that moved moves the pose too
    dc, dp = co.assert_matches(gi, gx, gp, ri, rx, rp, what)
    _worst["corner"] = max(_worst["corner"], dc)
    _worst["pose"] = max(_worst["pose"], dp)
    _worst["corners"] += len(ri)
    _worst["identical"] += int(np.sum(np.all(gx == rx, axis=1))) if len(ri) else 0
    return gi, gp


# ---- layout ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("legacy", [False, True])
def test_layout_matches_cv2(legacy):
    rng = np.random.default_rng(int(legacy))
    for sx in range(2, 13):
        for sy in range(2, 10):
            ids = None if (sx + sy) % 3 else rng.permutation(250)[: sx * sy // 2]
            ours = charuco_board((sx, sy), 0.037, 0.0271, ids, legacy)
            ref = co.cv_board((sx, sy), 0.037, 0.0271, ids, legacy)
            assert np.array_equal(ours.obj_points, np.array(ref.getObjPoints(), np.float32).reshape(-1, 4, 3)), (sx, sy)
            assert np.array_equal(ours.chessboard_corners, np.array(ref.getChessboardCorners(), np.float32).reshape(-1, 3)), (sx, sy)
            assert np.array_equal(ours.ids, ref.getIds().reshape(-1))
            # the harness's layout (the one fid_set_charuco_boards uploads) is the same
            obj = np.zeros((sx * sy // 2, 4, 3), np.float32)
            ch = np.zeros((ours.n_corners, 3), np.float32)
            nn, ni, ncn = np.zeros(ours.n_corners, np.int32), np.zeros((ours.n_corners, 2), np.int32), np.zeros((ours.n_corners, 2), np.int32)
            assert _load().hs_charuco_layout(sx, sy, C.c_float(0.037), C.c_float(0.0271), int(legacy), _p(obj), _p(ch), _p(nn), _p(ni), _p(ncn)) == 1
            assert np.array_equal(obj, ours.obj_points) and np.array_equal(ch, ours.chessboard_corners) and np.all(nn == 2)


def test_board_validation():
    for bad in (((1, 5), 0.04, 0.03), ((5, 5), 0.04, 0.05), ((5, 5), 0.04, 0.03, [1] * 12), ((34, 34), 0.04, 0.03)):
        with pytest.raises(ValueError):
            charuco_board(*bad)


# ---- detectBoard ------------------------------------------------------------------------------------------------------------------
W, H = 640, 480
K_SYN, D_REF = synth.camera_for(W, H)
D_ZERO = np.zeros(5)


def scene(rng, kind, size=None, legacy=False, ids=None, blur=True, min_markers=2, check_markers=True):
    sx, sy = size if size else (int(rng.integers(3, 9)), int(rng.integers(3, 8)))
    if isinstance(ids, str):  # "perm": a random subset of the dictionary
        ids = rng.permutation(250)[: sx * sy // 2]
    board = charuco_board((sx, sy), 0.04, 0.03, ids, legacy, min_markers, check_markers)
    cvb = cv_of(board)
    R, t = co.board_pose_in_view(cvb, rng, K_SYN, W, H, kind=kind)
    g = np.full((H, W), 128, np.uint8)
    co.render(g, cvb, R, t, K_SYN)
    return board, cvb, R, t, co.blur_noise(g, rng, blur)


@pytest.mark.parametrize("camera", ["none", "D_zero", "D_ref"])
@pytest.mark.parametrize("seed", range(3))
def test_detect_board(seed, camera):
    """Rendered boards at near, oblique and far views, subsets of the markers down to one, 0 - 0.5 px of marker corner noise, shuffled order,
    repeated detections and foreign ids; with a camera (both distortion models) and without."""
    rng = np.random.default_rng(100 + seed)
    K, D = (None, None) if camera == "none" else (K_SYN, D_ZERO if camera == "D_zero" else D_REF)
    for k in range(8):
        board, cvb, R, t, g = scene(rng, ["near", "oblique", "far"][k % 3], legacy=k % 4 == 3, ids=None if k % 3 else "perm")
        nm = len(board.ids)
        keep = None if k % 2 else sorted(rng.choice(nm, int(rng.integers(1, nm + 1)), replace=False).tolist())
        ids, corners = co.marker_detections(cvb, R, t, K_SYN, D_ZERO if D is None else D, rng, noise=float(rng.uniform(0, 0.5)), keep=keep,
                                            extra_ids=[251, 400][: k % 3], repeat=k % 2)
        check(board, g, ids, corners, K, D, "seed %d case %d" % (seed, k))


def test_single_marker_and_border():
    rng = np.random.default_rng(7)
    for k in range(6):
        board, cvb, R, t, g = scene(rng, "near", size=(5, 4))
        ids, corners = co.marker_detections(cvb, R, t, K_SYN, D_ZERO, rng, keep=[int(rng.integers(len(board.ids)))])
        for mm in (0, 1, 2):
            b = charuco_board((5, 4), 0.04, 0.03, min_markers=mm)
            for K in (None, K_SYN):
                check(b, g, ids, corners, K, D_ZERO, "single %d mm %d" % (k, mm))
    # a board partly outside the frame: corners within 2 px of the border are dropped
    board, cvb, R, t, g = scene(rng, "near", size=(8, 6))
    t = t + R @ np.array([0.12, 0.0, 0.0])
    g = np.full((H, W), 128, np.uint8)
    co.render(g, cvb, R, t, K_SYN)
    ids, corners = co.marker_detections(cvb, R, t, K_SYN, D_ZERO, rng)
    inside = np.all((corners >= 0) & (corners < [W, H]), axis=(1, 2))
    for K in (None, K_SYN):
        check(board, g, ids[inside], corners[inside], K, D_ZERO, "border")


def test_legacy_mismatch_and_check_markers():
    """A board rendered with the legacy pattern, detected as the default pattern: checkMarkers rejects it (no corner, status -3);
    with checkMarkers off every interpolated corner comes back.  Offset ids behave the same."""
    rng = np.random.default_rng(9)
    for ids in (None, np.arange(100, 124)):
        legacy = charuco_board((6, 8), 0.04, 0.03, ids, legacy=True)
        cvl = cv_of(legacy)
        R, t = co.board_pose_in_view(cvl, rng, K_SYN, W, H, kind="near")
        g = np.full((H, W), 128, np.uint8)
        co.render(g, cvl, R, t, K_SYN)
        g = co.blur_noise(g, rng)
        mids, mcs = co.marker_detections(cvl, R, t, K_SYN, D_ZERO, rng)
        for K in (None, K_SYN):
            on = charuco_board((6, 8), 0.04, 0.03, ids, legacy=False)
            gi, gp = check(on, g, mids, mcs, K, D_ZERO, "mismatch on")
            assert len(gi) == 0 and gp["status"] == -3
            off = charuco_board((6, 8), 0.04, 0.03, ids, legacy=False, check_markers=False)
            gi, _ = check(off, g, mids, mcs, K, D_ZERO, "mismatch off")
            assert len(gi) > 0


def test_collinear_corners_have_no_pose():
    """A 2 x N board has one row of corners: collinear, status -2 with a camera."""
    rng = np.random.default_rng(11)
    board, cvb, R, t, g = scene(rng, "near", size=(7, 2))
    ids, corners = co.marker_detections(cvb, R, t, K_SYN, D_ZERO, rng)
    gi, gp = check(board, g, ids, corners, K_SYN, D_ZERO, "collinear")
    assert len(gi) >= 4 and gp["status"] == -2


# ---- cornerSubPix with the ChArUco windows ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("win", range(1, 11))
def test_corner_subpix_windows(win):
    rng = np.random.default_rng(win)
    board, cvb, R, t, g = scene(rng, "near", size=(8, 6))
    proj = co.project(np.array(cvb.getChessboardCorners()), R, t, K_SYN, D_ZERO).astype(np.float32)
    pts = (proj + rng.uniform(-0.7, 0.7, proj.shape)).astype(np.float32)
    pts = pts[np.all((pts > 30) & (pts < [W - 30, H - 30]), axis=1)]
    ours = pts.copy()
    _load().hs_charuco_subpix(_p(g), W, H, _p(ours), len(ours), win, co.REFINE_MAX_ITER, C.c_double(co.REFINE_MIN_ACC))
    crit = (cv2.TERM_CRITERIA_MAX_ITER | cv2.TERM_CRITERIA_EPS, co.REFINE_MAX_ITER, co.REFINE_MIN_ACC)
    ref = cv2.cornerSubPix(g, pts.reshape(-1, 1, 2).copy(), (win, win), (0, 0), crit).reshape(-1, 2)
    # random starts up to 0.7 px off the corner: with small windows a few walks leave the corner's basin through nearly flat
    # patches, where the iteration is chaotic and a last-bit difference ends elsewhere; all others are bit-identical
    same = np.all(ours == ref, axis=1)
    print("window %d: %d of %d points bit-identical" % (win, same.sum(), len(same)))
    assert (~same).sum() <= 2
