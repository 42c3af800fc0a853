"""Recovery of missed board markers (fiducials_b200/csrc/marker_refine.cuh, compiled for the host from
tests/hostsim/marker_refine_hostsim.cpp) against cv2.aruco.ArucoDetector.refineDetectedMarkers on cv2's own detected and rejected
lists.  CPU only."""
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
from fiducials_b200.board import charuco_board, grid_board
from oracle import aruco_oracle as ao
import marker_refine_oracle as mo

_HERE = os.path.dirname(os.path.abspath(__file__))
_harness = None


def _load():
    """g++ build of the harness into a temporary directory (the tree may be read-only), once per session, without FMA contraction
    like the device build."""
    global _harness
    if _harness is None:
        tmp = tempfile.mkdtemp(prefix="fid_marker_refine_hostsim_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "libfid_marker_refine_hostsim.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, os.path.join(_HERE, "hostsim", "marker_refine_hostsim.cpp")])
        _harness = C.CDLL(so)
    return _harness


_vp = C.c_void_p


def _p(a):
    return None if a is None else a.ctypes.data_as(_vp)


P = ao.REFERENCE_PARAMS


def hs_refine(gray, boards, ids, corners, rej, K=None, D=None, refine=(10.0, 3.0, True), method=1, rel_win=100.0):
    """marker_refine.cuh on the host: ids, corners, remaining rejected list, recovered indices and boards, per-board status."""
    gray = np.ascontiguousarray(gray, np.uint8)
    H, W = gray.shape
    cap = len(ids) + sum(len(b.ids) for b in boards) + 1
    oi = np.zeros(cap, np.int32)
    oc = np.zeros((cap, 8), np.float32)
    oi[: len(ids)] = ids
    oc[: len(ids)] = np.asarray(corners, np.float32).reshape(-1, 8)
    rj = np.ascontiguousarray(np.asarray(rej, np.float32).reshape(-1, 8))
    bn = np.array([len(b.ids) for b in boards], np.int32)
    bids = np.ascontiguousarray(np.concatenate([np.asarray(b.ids, np.int32) for b in boards]))
    bobj = np.ascontiguousarray(np.concatenate([np.asarray(b.obj_points, np.float32).reshape(-1, 12) for b in boards]))
    Ka = None if K is None else np.ascontiguousarray(K, np.float64).reshape(9)
    Da = None if K is None else np.ascontiguousarray(D, np.float64).reshape(-1)[:5]
    ri, rb, st = np.zeros(cap, np.int32), np.zeros(cap, np.int32), np.zeros(len(boards), np.int32)
    n = _load().hs_refine(_p(gray), W, H, mo.DICT, method, P["cornerRefinementWinSize"], P["cornerRefinementMaxIterations"],
                          C.c_double(P["cornerRefinementMinAccuracy"]), C.c_double(rel_win), C.c_float(refine[0]), C.c_float(refine[1]),
                          int(refine[2]), len(boards), _p(bn), _p(bids), _p(bobj), _p(Ka), _p(Da), len(ids), _p(oi), _p(oc), cap, len(rj), _p(rj),
                          _p(ri), _p(rb), _p(st))
    assert n >= 0, n
    nr = n - len(ids)
    taken = set(ri[:nr].tolist())
    left = np.array([r for k, r in enumerate(rj) if k not in taken], np.float32).reshape(-1, 4, 2)
    return oi[:n].copy(), oc[:n].reshape(-1, 4, 2).copy(), left, ri[:nr].tolist(), rb[:nr].tolist(), st


_worst = {"subpix": 0.0, "recovered": 0, "cases": 0}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nmarker refinement vs cv2: %d cases, %d markers recovered, max |d corner| after cornerSubPix = %.3g px"
          % (_worst["cases"], _worst["recovered"], _worst["subpix"]))


def check(gray, boards, ids, corners, rej, K=None, D=None, refine=(10.0, 3.0, True), method=1, rel_win=100.0, what=""):
    """Ours against cv2 on the same lists: recovered ids and their order, recovered indices, boards and the remaining rejected list
    identical; corners bit-identical without cornerSubPix and within 1e-3 px with it; cv2 raises exactly where we skip a board."""
    det = mo.detector(refine, cornerRefinementMethod=method, relativeCornerRefinmentWinSize=rel_win)
    ri, rc, rr, rx, rb, raised = mo.refine(det, gray, boards, ids, corners, rej, K, D)
    gi, gc, gr, gx, gb, st = hs_refine(gray, boards, ids, corners, rej, K, D, refine, method, rel_win)
    assert [bool(s == -1) for s in st] == raised, (what, st, raised)
    assert gi.tolist() == ri.tolist(), (what, gi.tolist(), ri.tolist())
    assert gx == rx and gb == rb, (what, gx, rx, gb, rb)
    assert np.array_equal(gr, rr), what
    n0 = len(ids)
    assert np.array_equal(gc[:n0], rc[:n0]), what
    if method == 1:
        d = float(np.abs(gc[n0:] - rc[n0:]).max()) if len(gc) > n0 else 0.0
        _worst["subpix"] = max(_worst["subpix"], d)
        assert d <= 1e-3, (what, d)
    else:
        assert np.array_equal(gc[n0:], rc[n0:]), what
    _worst["cases"] += 1
    _worst["recovered"] += len(gx)
    return gx


W, H = 640, 480
K_SYN, D_REF = synth.camera_for(W, H)
D_ZERO = np.zeros(5)
BASE_METHOD = cv2.aruco.CORNER_REFINE_SUBPIX


def grid_scene(rng, size, kind, n_damaged=3, kinds=("stripe", "stripe", "full", "occlude"), blur=True, ids=None, length=0.04, sep=0.01):
    board = grid_board(size, length, sep, ids)
    R, t = mo.pose_in_view(board, rng, K_SYN, W, H, kind)
    g = np.full((H, W), 128, np.uint8)
    mo.render_grid(g, size, length, sep, R, t, K_SYN, ids)
    for k in rng.choice(len(board.ids), min(n_damaged, len(board.ids)), replace=False):
        mo.damage(g, board, int(k), R, t, K_SYN, rng, kinds[int(rng.integers(len(kinds)))])
    if blur:
        g = cv2.GaussianBlur(g, (3, 3), 0.8)
    return board, g


def charuco_scene(rng, size, kind, n_damaged=2):
    board = charuco_board(size, 0.04, 0.03)
    R, t = mo.pose_in_view(board, rng, K_SYN, W, H, kind)
    g = np.full((H, W), 128, np.uint8)
    mo.render_charuco(g, size, 0.04, 0.03, R, t, K_SYN)
    for k in rng.choice(len(board.ids), min(n_damaged, len(board.ids)), replace=False):
        mo.damage(g, board, int(k), R, t, K_SYN, rng, "stripe")
    return board, cv2.GaussianBlur(g, (3, 3), 0.8)


def lists(gray, method=BASE_METHOD):
    return mo.detect(mo.detector(cornerRefinementMethod=method), gray)


# ---- the premise and the main sweep --------------------------------------------------------------------------------------------
def test_damaged_grid_is_recovered():
    """A 5x4 grid with three markers' inner bits painted over: detection misses them, refinement gets them back (with and without a
    camera)."""
    rng = np.random.default_rng(1)
    board = grid_board((5, 4), 0.04, 0.01)
    R, t = mo.pose_in_view(board, rng, K_SYN, W, H, "near")
    g = np.full((H, W), 128, np.uint8)
    mo.render_grid(g, (5, 4), 0.04, 0.01, R, t, K_SYN)
    for k in (2, 7, 13):
        mo.damage(g, board, k, R, t, K_SYN, np.random.default_rng(k), "stripe")
    ids, corners, rej = lists(g)
    assert sorted(set(range(20)) - set(ids.tolist())) == [2, 7, 13]
    for K in (None, K_SYN):
        gx = check(g, [board], ids, corners, rej, K, D_ZERO, what="premise")
        assert len(gx) == 3


@pytest.mark.parametrize("camera", ["none", "D_zero", "D_ref"])
@pytest.mark.parametrize("seed", range(3))
def test_grid_boards(seed, camera):
    """Rendered GridBoards from 2x2 to 10x10 at near, far and oblique views with damaged, occluded and blurred markers."""
    rng = np.random.default_rng(10 + seed)
    K, D = (None, None) if camera == "none" else (K_SYN, D_ZERO if camera == "D_zero" else D_REF)
    for k in range(6):
        n = int(rng.integers(2, 11))
        size = (n, int(rng.integers(2, 11)))
        board, g = grid_scene(rng, size, ["near", "far", "oblique"][k % 3], n_damaged=int(rng.integers(1, 5)),
                              ids=None if k % 2 else rng.permutation(250)[: size[0] * size[1]])
        ids, corners, rej = lists(g)
        check(g, [board], ids, corners, rej, K, D, what="seed %d case %d %s" % (seed, k, size))


@pytest.mark.parametrize("refine", [(10.0, 3.0, True), (10.0, 3.0, False), (10.0, 0.0, True), (10.0, -1.0, True), (3.0, 3.0, True), (40.0, 3.0, True),
                                    (40.0, -1.0, False)])
def test_refine_parameters(refine):
    """checkAllOrders on and off, errorCorrectionRate -1, 0 and 3, several minRepDistance values."""
    rng = np.random.default_rng(20)
    for k in range(4):
        board, g = grid_scene(rng, (6, 5), ["near", "oblique"][k % 2], n_damaged=4)
        ids, corners, rej = lists(g)
        for K in (None, K_SYN):
            check(g, [board], ids, corners, rej, K, D_ZERO, refine, what="%s case %d" % (refine, k))


@pytest.mark.parametrize("method", [cv2.aruco.CORNER_REFINE_NONE, cv2.aruco.CORNER_REFINE_SUBPIX, cv2.aruco.CORNER_REFINE_CONTOUR])
@pytest.mark.parametrize("rel_win", [0.04, 0.3, 100.0])
def test_corner_methods(method, rel_win):
    """cornerSubPix only with CORNER_REFINE_SUBPIX, with the detector's window rule; NONE and CONTOUR keep the matched corners."""
    rng = np.random.default_rng(30)
    for k in range(3):
        board, g = grid_scene(rng, (5, 4), "near", n_damaged=3, kinds=("stripe",))
        ids, corners, rej = lists(g, method)
        check(g, [board], ids, corners, rej, K_SYN if k % 2 else None, D_ZERO, method=method, rel_win=rel_win, what="method %d case %d" % (method, k))


def test_two_boards_and_charuco():
    """A grid board and a ChArUco board in one frame, refined in sequence: the second call sees what the first recovered and took."""
    rng = np.random.default_rng(40)
    for k in range(4):
        grid = grid_board((4, 3), 0.03, 0.008, ids=np.arange(100, 112))
        ch = charuco_board((5, 4), 0.03, 0.022)
        g = np.full((H, W), 128, np.uint8)
        Rg, tg = mo.pose_in_view(grid, rng, K_SYN, W, H, "far")
        tg = tg + np.array([-0.08, 0.0, 0.0])
        Rc, tc = mo.pose_in_view(ch, rng, K_SYN, W, H, "far")
        tc = tc + np.array([0.08, 0.0, 0.0])
        mo.render_grid(g, (4, 3), 0.03, 0.008, Rg, tg, K_SYN, np.arange(100, 112))
        mo.render_charuco(g, (5, 4), 0.03, 0.022, Rc, tc, K_SYN)
        for kk in rng.choice(12, 2, replace=False):
            mo.damage(g, grid, int(kk), Rg, tg, K_SYN, rng, "stripe")
        for kk in rng.choice(10, 2, replace=False):
            mo.damage(g, ch, int(kk), Rc, tc, K_SYN, rng, "stripe")
        g = cv2.GaussianBlur(g, (3, 3), 0.8)
        ids, corners, rej = lists(g)
        for K in (None, K_SYN):
            for boards in ([grid, ch], [ch, grid]):
                check(g, boards, ids, corners, rej, K, D_ZERO, what="two boards %d" % k)
        # the same board twice: the second call has nothing left to recover
        check(g, [ch, ch], ids, corners, rej, K_SYN, D_ZERO, what="twice %d" % k)


def test_edge_cases():
    """No detections, no rejected candidates, no board marker detected, a repeated detection, and a non-planar board with and
    without a camera (cv2 raises; nothing is recovered)."""
    rng = np.random.default_rng(50)
    board, g = grid_scene(rng, (5, 4), "near", n_damaged=3, kinds=("stripe",))
    ids, corners, rej = lists(g)
    for K in (None, K_SYN):
        assert check(g, [board], ids[:0], corners[:0], rej, K, D_ZERO, what="no detections") == []
        assert check(g, [board], ids, corners, rej[:0], K, D_ZERO, what="no rejected") == []
        other = grid_board((3, 3), 0.04, 0.01, ids=np.arange(200, 209))
        assert check(g, [other], ids, corners, rej, K, D_ZERO, what="no board marker") == []
        rep_ids = np.concatenate([ids, ids[:1]])
        rep_c = np.concatenate([corners, corners[:1] + 0.3]).astype(np.float32)
        check(g, [board], rep_ids, rep_c, rej, K, D_ZERO, what="repeated")
        # a board whose points are not on one plane: without a camera cv2 asserts; with one, solvePnP raises below 6 points
        obj = board.obj_points.copy()
        obj[:, 2, 2] = np.float32(0.01)  # one corner of every marker lifted: even one marker's points are not planar
        bent = type(board)(board.ids, obj)
        one = ids[:1], corners[:1]
        check(g, [bent], one[0], one[1], rej, K, D_ZERO, what="non-planar, one marker")
        check(g, [bent], ids, corners, rej, K, D_ZERO, what="non-planar")
        assert hs_refine(g, [bent], one[0], one[1], rej, K, D_ZERO)[5].tolist() == [-1]
    assert hs_refine(g, [bent], ids, corners, rej)[5].tolist() == [-1]
