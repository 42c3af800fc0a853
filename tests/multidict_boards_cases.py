"""Boards bound to dictionary families (fid_set_family_boards, fid_set_family_charuco_boards, fid_set_family_diamonds): seeded
frames in which several families carry the same raw ids, and the cv2 4.13 composition a user writes for them.  Used by
tests/test_multidict_boards_oracle.py (CPU) and tests/test_gpu_multidict_boards.py.  TEST INFRASTRUCTURE ONLY.

Per frame: ``corners, ids, _, di = ArucoDetector(dicts, params).detectMarkersMultiDict(img)``; a board bound to family k then sees
``corners[di == k], ids[di == k]`` alone, in list order.
"""
from __future__ import annotations

import cv2
import numpy as np

from fiducials_b200.board import CharucoBoard, grid_board
from oracle import aruco_oracle as ao

A = cv2.aruco
W, H = 1280, 720
GRID_MARKER, GRID_SEP = 0.05, 0.015           # metres: 2 x 2 GridBoards, 110 px markers
GRID_PX, GRID_SEP_PX = 110, 33
CH_SIZE, CH_SQUARE, CH_MARKER = (5, 4), 0.04, 0.03   # the ChArUco board, 80 px squares
CH_PX = 80
DIA_SQUARE, DIA_MARKER = 0.04, 0.025           # the diamonds, 64 px squares
DIA_PX = 64
DIA_IDS = (20, 21, 22, 23)


def cv_dict(d):
    return A.getPredefinedDictionary(d)


def _paste(g, img, x, y):
    g[y:y + img.shape[0], x:x + img.shape[1]] = img


def _grid_image(d, ids):
    b = A.GridBoard((2, 2), GRID_MARKER, GRID_SEP, cv_dict(d), np.asarray(ids, np.int32))
    m = GRID_PX // 3
    side = 2 * GRID_PX + GRID_SEP_PX + 2 * m
    return b.generateImage((side, side), marginSize=m, borderBits=1)


def _charuco_image(d, size, square_px, ids=None):
    b = A.CharucoBoard(tuple(size), 1.0, CH_MARKER / CH_SQUARE if size != (3, 3) else DIA_MARKER / DIA_SQUARE, cv_dict(d),
                       None if ids is None else np.asarray(ids, np.int32))
    m = square_px // 3
    return b.generateImage((size[0] * square_px + 2 * m, size[1] * square_px + 2 * m), marginSize=m, borderBits=1)


def _finish(g, rng):
    """A mild random perspective warp of the whole frame, blur and noise (as multidict_oracle.render_mixed)."""
    Hm = np.array([[1 + rng.uniform(-0.03, 0.03), rng.uniform(-0.05, 0.05), rng.uniform(-5, 5)],
                   [rng.uniform(-0.05, 0.05), 1 + rng.uniform(-0.03, 0.03), rng.uniform(-5, 5)],
                   [rng.uniform(-2e-5, 2e-5), rng.uniform(-2e-5, 2e-5), 1.0]])
    g = cv2.warpPerspective(g, Hm, (W, H), flags=cv2.INTER_LINEAR, borderValue=200)
    g = cv2.GaussianBlur(g, (3, 3), 0.7)
    g = np.clip(g + rng.normal(0, 2.0, g.shape), 0, 255).astype(np.uint8)
    return np.ascontiguousarray(cv2.cvtColor(g, cv2.COLOR_GRAY2BGR))


def render_grids(seed, dicts=(A.DICT_4X4_50, A.DICT_5X5_1000)):
    """Two 2 x 2 GridBoards with ids 0..3, one per family in dicts: every raw id is on the frame twice."""
    rng = np.random.default_rng(seed)
    g = np.full((H, W), 200, np.uint8)
    _paste(g, _grid_image(dicts[0], range(4)), 80 + int(rng.integers(0, 60)), 120 + int(rng.integers(0, 60)))
    _paste(g, _grid_image(dicts[1], range(4)), 700 + int(rng.integers(0, 60)), 160 + int(rng.integers(0, 60)))
    return _finish(g, rng)


def render_mixed_boards(seed):
    """DICT_6X6_250: a 5 x 4 ChArUco board with ids 0..9 and a diamond with ids DIA_IDS; AprilTag 36h11: a 5 x 2 GridBoard-like row of
    tags 0..9 and a look-alike diamond with the same ids; DICT_4X4_50: a 2 x 2 GridBoard with ids 0..3."""
    rng = np.random.default_rng(seed)
    g = np.full((H, W), 200, np.uint8)
    j = lambda: int(rng.integers(0, 20))  # noqa: E731
    _paste(g, _charuco_image(A.DICT_6X6_250, CH_SIZE, CH_PX), 30 + j(), 20 + j())
    tags = A.GridBoard((5, 2), 0.04, 0.012, cv_dict(A.DICT_APRILTAG_36h11), np.arange(10, dtype=np.int32)).generateImage((520, 220), marginSize=20, borderBits=1)
    _paste(g, tags, 30 + j(), 440 + j())
    _paste(g, _grid_image(A.DICT_4X4_50, range(4)), 540 + j(), 20 + j())
    _paste(g, _charuco_image(A.DICT_6X6_250, (3, 3), DIA_PX, DIA_IDS), 590 + j(), 420 + j())
    _paste(g, _charuco_image(A.DICT_APRILTAG_36h11, (3, 3), DIA_PX, DIA_IDS), 900 + j(), 380 + j())
    return _finish(g, rng)


def grid(ids=range(4)):
    return grid_board((2, 2), GRID_MARKER, GRID_SEP, list(ids))


def tags():
    """The AprilTag row of render_mixed_boards as a board."""
    return grid_board((5, 2), 0.04, 0.012, list(range(10)))


def charuco():
    return CharucoBoard(CH_SIZE, CH_SQUARE, CH_MARKER)


def cv2_multi(bgr, dicts, method=1, inverted=False):
    """detectMarkersMultiDict with the reference parameters: ids [n], corners [n, 4, 2] float32, dict indices [n]."""
    p = ao.reference_detector_params(cornerRefinementMethod=method)
    p.detectInvertedMarker = bool(inverted)
    det = A.ArucoDetector(cv_dict(dicts[0]), p)
    det.setDictionaries([cv_dict(d) for d in dicts])
    corners, ids, _, di = det.detectMarkersMultiDict(bgr)
    if ids is None or len(ids) == 0:
        return np.zeros(0, np.int32), np.zeros((0, 4, 2), np.float32), np.zeros(0, np.int32)
    return ids.reshape(-1).astype(np.int32), np.array(corners, np.float32).reshape(-1, 4, 2), np.asarray(di).reshape(-1).astype(np.int32)


def cv2_single(bgr, d, method=1, inverted=False):
    p = ao.reference_detector_params(cornerRefinementMethod=method)
    p.detectInvertedMarker = bool(inverted)
    corners, ids, _ = A.ArucoDetector(cv_dict(d), p).detectMarkers(bgr)
    if ids is None or len(ids) == 0:
        return np.zeros(0, np.int32), np.zeros((0, 4, 2), np.float32)
    return ids.reshape(-1).astype(np.int32), np.array(corners, np.float32).reshape(-1, 4, 2)


def family(ids, corners, di, k):
    """corners[di == k], ids[di == k] in list order: what a stage bound to family k sees."""
    sel = np.asarray(di) == k
    return np.asarray(ids)[sel], np.asarray(corners, np.float32).reshape(-1, 4, 2)[sel]


def cv_charuco(board: CharucoBoard, d):
    """cv2.aruco.CharucoBoard of a fiducials_b200 CharucoBoard in family dictionary d."""
    b = A.CharucoBoard(tuple(board.size), board.square_length, board.marker_length, cv_dict(d), np.asarray(board.ids, np.int32))
    b.setLegacyPattern(bool(board.legacy))
    return b


def diamond_detector(d, K=None, D=None, method=1, min_markers=2, check_markers=True):
    """CharucoDetector(CharucoBoard((3, 3), square, marker, dicts[k]), ...) with the reference parameters."""
    cp = A.CharucoParameters()
    if K is not None:
        cp.cameraMatrix = np.asarray(K, np.float64).reshape(3, 3)
        cp.distCoeffs = np.asarray(D, np.float64).reshape(1, -1)
    cp.minMarkers = int(min_markers)
    cp.checkMarkers = bool(check_markers)
    return A.CharucoDetector(A.CharucoBoard((3, 3), DIA_SQUARE, DIA_MARKER, cv_dict(d)), cp, ao.reference_detector_params(cornerRefinementMethod=method))
