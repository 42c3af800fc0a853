"""Marker boards for fid_set_boards / fid_estimate_board_poses: a known rigid layout of markers whose pose is solved from the corners
of every visible marker in one cv::solvePnP (SOLVEPNP_ITERATIVE), as cv::aruco::Board::matchImagePoints + solvePnP compute it."""
from __future__ import annotations

from typing import Iterable, Optional, Sequence, Tuple

import numpy as np


class Board:
    """A rigid set of markers: ``ids`` [n] (distinct) and ``obj_points`` [n][4][3] in metres, each marker's corners in the order
    the detector reports them (cv::aruco::Board's order: top-left, top-right, bottom-right, bottom-left as the marker is printed).
    The points are kept as float32, as cv::aruco::Board stores them."""

    def __init__(self, ids: Iterable[int], obj_points):
        self.ids = np.ascontiguousarray(np.asarray(list(ids) if not isinstance(ids, np.ndarray) else ids, np.int64).reshape(-1)).astype(np.int32)
        self.obj_points = np.ascontiguousarray(np.asarray(obj_points, np.float32).reshape(-1, 4, 3))
        if len(self.ids) != len(self.obj_points):
            raise ValueError("Board: %d ids but %d markers of object points" % (len(self.ids), len(self.obj_points)))
        if not 1 <= len(self.ids) <= 4096:
            raise ValueError("Board: 1..4096 markers, got %d" % len(self.ids))
        if len(np.unique(self.ids)) != len(self.ids):
            raise ValueError("Board: repeated marker id")
        if not np.all(np.isfinite(self.obj_points)):
            raise ValueError("Board: non-finite object point")

    def __len__(self):
        return len(self.ids)

    def __repr__(self):
        return "Board(%d markers, ids %s)" % (len(self.ids), self.ids[:8].tolist() + (["..."] if len(self.ids) > 8 else []))


def grid_board(size: Tuple[int, int], marker_length: float, separation: float, ids: Optional[Sequence[int]] = None) -> Board:
    """The layout of cv::aruco::GridBoard(size, markerLength, markerSeparation, dictionary, ids) of OpenCV 4.13: size = (columns,
    rows); marker k sits at column k % columns, row k // columns, its top-left corner at (col, row) * (length + separation) with y
    growing down the board, corners TL, TR, BR, BL; ids default to 0 .. columns * rows - 1.  The arithmetic is float32, as there."""
    w, h = int(size[0]), int(size[1])
    if w <= 0 or h <= 0 or not marker_length > 0 or not separation > 0:
        raise ValueError("grid_board: size, marker_length and separation must be positive (as cv::aruco::GridBoard requires)")
    n = w * h
    ids = np.arange(n) if ids is None else np.asarray(ids).reshape(-1)
    if len(ids) != n:
        raise ValueError("grid_board: %d ids for %d markers" % (len(ids), n))
    L, s = np.float32(marker_length), np.float32(separation)
    step = np.float32(L + s)
    obj = np.zeros((n, 4, 3), np.float32)
    for k in range(n):
        x0, y0 = np.float32(np.float32(k % w) * step), np.float32(np.float32(k // w) * step)
        obj[k] = [[x0, y0, 0], [np.float32(x0 + L), y0, 0], [np.float32(x0 + L), np.float32(y0 + L), 0], [x0, np.float32(y0 + L), 0]]
    return Board(ids, obj)


class CharucoBoard:
    """A ChArUco board as fid_set_charuco_boards takes it, with its layout (cv::aruco::CharucoBoard of OpenCV 4.13): ``obj_points``
    [n_markers][4][3] and ``chessboard_corners`` [n_corners][3], float32, equal to cv2's getObjPoints() / getChessboardCorners()."""

    def __init__(self, size, square_length, marker_length, ids=None, legacy=False, min_markers=2, check_markers=True):
        sx, sy = int(size[0]), int(size[1])
        if sx < 2 or sy < 2 or (sx - 1) * (sy - 1) > 1024:
            raise ValueError("charuco_board: size must be >= 2 x 2 with at most 1024 chessboard corners")
        if not 0 < marker_length < square_length:
            raise ValueError("charuco_board: 0 < marker_length < square_length")
        if min_markers not in (0, 1, 2):
            raise ValueError("charuco_board: min_markers must be 0, 1 or 2")
        n = sx * sy // 2
        self.size, self.legacy = (sx, sy), bool(legacy)
        self.square_length, self.marker_length = float(np.float32(square_length)), float(np.float32(marker_length))
        self.ids = np.arange(n, dtype=np.int32) if ids is None else np.ascontiguousarray(np.asarray(ids).reshape(-1), np.int32)
        if len(self.ids) != n or len(np.unique(self.ids)) != n:
            raise ValueError("charuco_board: %d distinct ids needed" % n)
        self.min_markers, self.check_markers = int(min_markers), bool(check_markers)
        S, L = np.float32(square_length), np.float32(marker_length)
        diff = np.float32((S - L) / np.float32(2))
        obj = []
        for y in range(sy):
            for x in range(sx):
                if (legacy and sy % 2 == 0 and (y + 1) % 2 == x % 2) or (not (legacy and sy % 2 == 0) and y % 2 == x % 2):
                    continue
                x0, y0 = np.float32(np.float32(x) * S + diff), np.float32(np.float32(y) * S + diff)
                obj.append([[x0, y0, 0], [np.float32(x0 + L), y0, 0], [np.float32(x0 + L), np.float32(y0 + L), 0], [x0, np.float32(y0 + L), 0]])
        self.obj_points = np.array(obj, np.float32).reshape(-1, 4, 3)
        self.chessboard_corners = np.array([[np.float32(x + 1) * S, np.float32(y + 1) * S, 0] for y in range(sy - 1) for x in range(sx - 1)], np.float32)

    @property
    def n_corners(self):
        return (self.size[0] - 1) * (self.size[1] - 1)

    def __repr__(self):
        return "CharucoBoard(%dx%d, %d corners)" % (self.size[0], self.size[1], self.n_corners)


def charuco_board(size, square_length, marker_length, ids=None, legacy=False, min_markers=2, check_markers=True) -> CharucoBoard:
    """cv::aruco::CharucoBoard(size, squareLength, markerLength, dictionary, ids) with setLegacyPattern(legacy), and the
    CharucoParameters minMarkers / checkMarkers its detection uses.  size = (columns, rows) of squares."""
    return CharucoBoard(size, square_length, marker_length, ids, legacy, min_markers, check_markers)
