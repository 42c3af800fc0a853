"""One pose per marker board (fiducials_b200/csrc/board_pnp.cuh, compiled for the host from tests/hostsim/board_hostsim.cpp) against
cv2.aruco.Board.matchImagePoints + cv2.solvePnP(SOLVEPNP_ITERATIVE), and the grid layout of fiducials_b200.board against
cv2.aruco.GridBoard.  CPU only."""
import atexit
import ctypes as C
import math
import os
import shutil
import subprocess
import tempfile

import cv2
import numpy as np
import pytest

from fiducials_b200 import synth
from fiducials_b200.board import Board, grid_board
import board_oracle as bo

_HERE = os.path.dirname(os.path.abspath(__file__))
_harness = None


def _load():
    """g++ build of the harness into a temporary directory (the tree may be read-only), once per session; the flags of
    tests/hostsim/build.sh (no FMA contraction, like the device build)."""
    global _harness
    if _harness is None:
        tmp = tempfile.mkdtemp(prefix="fid_board_hostsim_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "libfid_board_hostsim.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, os.path.join(_HERE, "hostsim", "board_hostsim.cpp")])
        _harness = C.CDLL(so)
    return _harness


K_SYN, D_REF = synth.camera_for(640, 480)
D_ZERO = np.zeros(5)
_vp = C.c_void_p


def _p(a):
    return a.ctypes.data_as(_vp)


def hs_match(board, ids, corners):
    ids = np.ascontiguousarray(ids, np.int32).reshape(-1)
    corners = np.ascontiguousarray(corners, np.float32).reshape(-1, 8)
    n = len(ids)
    obj = np.zeros((4 * n + 1, 3), np.float32)
    img = np.zeros((4 * n + 1, 2), np.float32)
    m = _load().hs_board_match(n, _p(ids), _p(corners), len(board), _p(board.ids), _p(board.obj_points), _p(obj), _p(img))
    return obj[: 4 * m], img[: 4 * m]


def hs_board_pose(board, ids, corners, K, D):
    """board_pnp.cuh on the host: a dict like board_oracle.board_pose."""
    ids = np.ascontiguousarray(ids, np.int32).reshape(-1)
    corners = np.ascontiguousarray(corners, np.float32).reshape(-1, 8)
    K = np.ascontiguousarray(K, np.float64).reshape(9)
    D = np.ascontiguousarray(D, np.float64).reshape(-1)[:5]
    out = np.zeros(20)
    _load().hs_board_pose(len(ids), _p(ids), _p(corners), len(board), _p(board.ids), _p(board.obj_points), _p(K), _p(D), _p(out))
    return dict(status=int(out[0]), n_markers=int(out[1]), n_points=int(out[2]), rvec=out[3:6].copy(), tvec=out[6:9].copy(), rotation=out[9:13].copy(),
                image_error=float(out[13]), lm_iters=int(out[14]))


_worst = {"pose": 0.0, "image_error": 0.0}


def _check(cases, K, D, tol=bo.TOL):
    n_pose = 0
    for i, (b, ids, corners) in enumerate(cases):
        got = hs_board_pose(b, ids, corners, K, D)
        ref = bo.board_pose(b, ids, corners, K, D)
        dp, de = bo.assert_matches(got, ref, "case %d" % i, tol)
        _worst["pose"] = max(_worst["pose"], dp)
        _worst["image_error"] = max(_worst["image_error"], de)
        n_pose += got["status"] == 1
    return n_pose


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nboard pose vs cv2: max |d rvec|,|d tvec| = %.3g, max relative d image_error = %.3g" % (_worst["pose"], _worst["image_error"]))


# ---- the grid layout ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("size,length,sep,ids", [((2, 2), 0.04, 0.01, None), ((5, 7), 0.033, 0.0071, None), ((10, 3), 0.1, 0.02, "perm"),
                                                 ((1, 6), 0.0125, 0.001, None), ((4, 4), 0.07, 0.35, "perm")])
def test_grid_board_matches_cv2(size, length, sep, ids):
    n = size[0] * size[1]
    if ids == "perm":
        ids = np.random.default_rng(n).permutation(250)[:n]
    ours = grid_board(size, length, sep, ids)
    ref = cv2.aruco.GridBoard(size, length, sep, bo.DICT, None if ids is None else np.asarray(ids, np.int32))
    assert np.array_equal(ours.obj_points, np.array(ref.getObjPoints(), np.float32).reshape(-1, 4, 3))
    assert np.array_equal(ours.ids, ref.getIds().reshape(-1))


def test_board_validation():
    for bad in (([1, 1], np.zeros((2, 4, 3))), ([1], np.full((1, 4, 3), np.nan)), ([], np.zeros((0, 4, 3))), ([1, 2], np.zeros((1, 4, 3)))):
        with pytest.raises(ValueError):
            Board(*bad)


# ---- matching -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(6))
def test_match_equals_match_image_points(seed):
    rng = np.random.default_rng(seed)
    w, h = int(rng.integers(2, 8)), int(rng.integers(2, 8))
    b = grid_board((w, h), 0.05, 0.01, rng.permutation(250)[: w * h] if seed % 2 else None)
    R, t = bo.board_in_view(b, rng, K_SYN)
    keep = sorted(rng.choice(len(b), int(rng.integers(1, len(b) + 1)), replace=False).tolist())
    ids, corners = bo.detections(b, R, t, K_SYN, D_REF, rng, keep=keep, extra_ids=[300, 251, 999][: seed % 4], repeat=seed % 3)
    obj, img = hs_match(b, ids, corners)
    ro, ri = bo.match(b, ids, corners)
    assert np.array_equal(obj, ro) and np.array_equal(img, ri)
    assert len(obj) == 4 * (len(keep) + seed % 3)


def test_match_empty_and_off_board():
    b = grid_board((3, 3), 0.05, 0.01)
    for ids in ([], [100, 200]):
        corners = np.zeros((len(ids), 4, 2), np.float32) + 50
        obj, img = hs_match(b, ids, corners)
        ro, ri = bo.match(b, ids, corners)
        assert len(obj) == len(ro) == 0
        got = hs_board_pose(b, ids, corners, K_SYN, D_REF)
        assert got["status"] == 0 and got["n_points"] == 0 and not np.any(got["rvec"]) and got["image_error"] == 0.0


# ---- the homography ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [4, 5, 8, 40, 400])
def test_homography_matches_find_homography(n):
    rng = np.random.default_rng(n)
    for _ in range(10):
        src = rng.uniform(-0.5, 0.5, (n, 2))
        H = np.array([[1.0, 0.1, 0.05], [-0.08, 0.9, -0.02], [0.3, -0.2, 1.0]]) + rng.normal(0, 0.05, (3, 3))
        dst = cv2.perspectiveTransform(src.reshape(-1, 1, 2), H).reshape(-1, 2) + rng.normal(0, 1e-3, (n, 2))
        ours = np.zeros(9)
        assert _load().hs_homography(n, _p(np.ascontiguousarray(src)), _p(np.ascontiguousarray(dst)), _p(ours)) == 1
        ref = cv2.findHomography(src, dst, 0)[0].reshape(9)
        assert np.abs(ours - ref).max() <= 1e-6 * np.abs(ref).max(), (ours, ref)


# ---- the pose ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [D_REF, D_ZERO], ids=["D_ref", "D_zero"])
@pytest.mark.parametrize("seed", range(4))
def test_grid_boards(seed, D):
    """GridBoards 2x2 .. 10x10 at near, far and oblique poses, subsets down to one marker, noise, ids off the board, repeats."""
    cases = bo.grid_cases(10 + seed, K_SYN, D, n=15)
    assert _check(cases, K_SYN, D) == len(cases)


@pytest.mark.parametrize("D", [D_REF, D_ZERO], ids=["D_ref", "D_zero"])
def test_single_marker_visible(D):
    rng = np.random.default_rng(3)
    cases = []
    for k in range(12):
        b = grid_board((4, 3), 0.05, 0.01)
        R, t = bo.board_in_view(b, rng, K_SYN, kind=["near", "far", "oblique"][k % 3])
        cases.append((b,) + bo.detections(b, R, t, K_SYN, D, rng, noise=0.3, keep=[int(rng.integers(len(b)))]))
    assert _check(cases, K_SYN, D) == len(cases)


@pytest.mark.parametrize("D", [D_REF, D_ZERO], ids=["D_ref", "D_zero"])
def test_tilted_plane_off_z0(D):
    """A planar board in a tilted plane with z != 0 (the plane-frame rotation Rt / Tt of the planar branch)."""
    rng = np.random.default_rng(21)
    cases = []
    for k in range(10):
        b = bo.transformed(grid_board((int(rng.integers(2, 6)), int(rng.integers(2, 6))), 0.05, 0.012), bo._rot(rng.normal(0, 0.6, 3)), rng.normal(0, 0.3, 3))
        R, t = bo.board_in_view(b, rng, K_SYN, kind=["near", "far", "oblique"][k % 3])
        keep = sorted(rng.choice(len(b), int(rng.integers(1, len(b) + 1)), replace=False).tolist())
        cases.append((b,) + bo.detections(b, R, t, K_SYN, D, rng, noise=float(rng.uniform(0, 0.5)), keep=keep))
    assert _check(cases, K_SYN, D) == len(cases)


@pytest.mark.parametrize("D", [D_REF, D_ZERO], ids=["D_ref", "D_zero"])
@pytest.mark.parametrize("faces", [2, 3])
def test_cube_faces_non_planar(faces, D):
    rng = np.random.default_rng(30 + faces)
    b = bo.cube_board(faces)
    cases = []
    for k in range(10):
        R = bo._rot([0.0, 0.0, 0.0]) @ bo._rot([rng.uniform(-0.5, -0.3), rng.uniform(-0.8, -0.4), rng.uniform(-0.3, 0.3)])
        t = np.array([rng.uniform(-0.1, 0.1), rng.uniform(-0.1, 0.1), rng.uniform(0.8, 2.0)])
        cases.append((b,) + bo.detections(b, R, t, K_SYN, D, rng, noise=float(rng.uniform(0, 0.5))))
    # every face but one hidden: one visible face is planar (the branch is chosen per frame)
    cases.append((b,) + bo.detections(b, R, t, K_SYN, D, rng, noise=0.2, keep=[1]))
    assert _check(cases, K_SYN, D) == len(cases)


@pytest.mark.parametrize("D", [D_REF, D_ZERO], ids=["D_ref", "D_zero"])
def test_four_non_coplanar_points_raise_in_cv2(D):
    """One marker whose 4 board corners are not coplanar: cv2.solvePnP raises (status -1); two of them (8 points) are solved."""
    rng = np.random.default_rng(40)
    b = bo.bent_marker()
    R, t = bo._rot([math.pi, 0.1, 0.0]), np.array([0.02, -0.01, 0.6])
    ids, corners = bo.detections(b, R, t, K_SYN, D, rng, noise=0.1)
    got, ref = hs_board_pose(b, ids, corners, K_SYN, D), bo.board_pose(b, ids, corners, K_SYN, D)
    assert ref["status"] == -1 and got["status"] == -1 and got["n_points"] == 4
    # slightly bent (below the planarity threshold): planar, solved
    flat = bo.bent_marker(bend=1e-5)
    ids, corners = bo.detections(flat, R, t, K_SYN, D, rng, noise=0.1)
    assert _check([(flat, ids, corners)], K_SYN, D) == 1
    # the bent marker detected twice: 8 non-planar points, enough for the DLT branch
    ids3, corners3 = bo.detections(b, R, t, K_SYN, D, rng, noise=0.1)
    ids3, corners3 = np.concatenate([ids3, ids3]), np.concatenate([corners3, corners3 + 0.2])
    assert _check([(b, ids3, corners3)], K_SYN, D) == 1
