"""Camera calibration on the GPU: cv2.calibrateCameraExtended for K and the plumb_bob coefficients k1 k2 p1 p2 k3
(fid_calibrate_camera, fiducials_b200/csrc/calib.cuh), cv2.calibrateCameraROExtended, which also re-estimates the board's points
(fid_calibrate_camera_ro), and the views a ChArUco detection gives them."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib

CALIB_USE_INTRINSIC_GUESS = 0x00001  # the values of cv2.CALIB_*
CALIB_FIX_ASPECT_RATIO = 0x00002
CALIB_FIX_PRINCIPAL_POINT = 0x00004
CALIB_ZERO_TANGENT_DIST = 0x00008
CALIB_FIX_FOCAL_LENGTH = 0x00010
CALIB_FIX_K1 = 0x00020
CALIB_FIX_K2 = 0x00040
CALIB_FIX_K3 = 0x00080

CALIB_STATUS = {1: "a view has fewer than 4 points (or more than 4096)", 2: "non-planar calibration rigs need an intrinsic guess",
                3: "a view's points give no homography (collinear?)", 4: "the intrinsic guess is out of range", 5: "a view's initial pose cannot be solved",
                6: "non-finite points or inconsistent sizes", 7: "releasing the object points needs views with the same object points",
                8: "the released system has a non-positive pivot", 9: "releasing leaves as many free parameters as residuals or more"}


class CalibError(_lib.FidError):
    """fid_calibrate_camera refused the input where cv2.calibrateCamera raises; .calib_status is the FID_CALIB_E_* code."""

    def __init__(self, status, calib_status):
        self.calib_status = calib_status
        super().__init__(status, CALIB_STATUS.get(calib_status, ""))


def _views(object_points, image_points):
    if len(object_points) != len(image_points):
        raise ValueError("calibrate_camera: as many object point sets as image point sets needed")
    obj = [np.ascontiguousarray(o, np.float32).reshape(-1, 3) for o in object_points]
    img = [np.ascontiguousarray(m, np.float32).reshape(-1, 2) for m in image_points]
    for o, m in zip(obj, img):
        if len(o) != len(m):
            raise ValueError("calibrate_camera: a view has different numbers of object and image points")
    off = np.zeros(len(obj) + 1, np.int32)
    off[1:] = np.cumsum([len(o) for o in obj])
    cat = lambda a, w: np.ascontiguousarray(np.concatenate(a) if a else np.zeros((0, w), np.float32), np.float32)
    return off, cat(obj, 3), cat(img, 2)


def _guess(K, D):
    if K is None and D is None:
        return None
    Kg = np.eye(3) if K is None else np.asarray(K, np.float64).reshape(3, 3)
    Dg = np.zeros(5) if D is None else np.asarray(D, np.float64).reshape(-1)
    if len(Dg) > 5 and np.any(Dg[5:] != 0):
        raise ValueError("calibrate_camera: only k1 k2 p1 p2 k3 (fid_camera) are supported")
    guess = _lib.fid_camera()
    for i in range(9):
        guess.K[i] = float(Kg.reshape(9)[i])
    for i in range(min(5, len(Dg))):
        guess.D[i] = float(Dg[i])
    return guess


def _run(fn, object_points, image_points, image_size, K, D, flags, criteria, device, stats, extra=()):
    lib = _lib.load()
    off, obj, img = _views(object_points, image_points)
    nv = len(off) - 1
    guess = _guess(K, D)
    crit = None
    if criteria is not None:
        crit = _lib.fid_calib_criteria(int(criteria[0]), int(criteria[1]), float(criteria[2]))
    res = _lib.fid_calib_result()
    rv, tv = np.zeros((max(nv, 1), 3)), np.zeros((max(nv, 1), 3))
    se, pve = np.zeros((max(nv, 1), 6)), np.zeros(max(nv, 1))
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    st = getattr(lib, fn)(int(device), nv, vp(off), vp(obj), vp(img), int(image_size[0]), int(image_size[1]), None if guess is None else C.byref(guess), int(flags),
                          None if crit is None else C.byref(crit), C.byref(res), vp(rv), vp(tv), vp(se), vp(pve), None if stats is None else C.byref(stats), *extra)
    if st == -1 and res.status:
        raise CalibError(st, res.status)
    _lib.check(st, fn)
    Kout = np.array(res.camera.K[:], np.float64).reshape(3, 3)
    Dout = np.array(res.camera.D[:], np.float64).reshape(1, 5)
    std_int = np.zeros((18, 1))
    std_int[:9, 0] = res.std_intrinsics[:]
    return (res.rms, Kout, Dout, tuple(r.reshape(3, 1).copy() for r in rv[:nv]), tuple(t.reshape(3, 1).copy() for t in tv[:nv]), std_int,
            se[:nv].reshape(-1, 1).copy(), pve[:nv].reshape(-1, 1).copy())


def calibrate_camera(object_points, image_points, image_size, K=None, D=None, flags=0, criteria=None, device=0, stats=None):
    """cv2.calibrateCameraExtended(object_points, image_points, image_size, K, D, flags=flags, criteria=criteria) on the GPU.

    object_points / image_points: per view [n][3] / [n][2] (float32, as cv2 takes them); image_size = (width, height).  K, D: the
    intrinsic guess (CALIB_USE_INTRINSIC_GUESS) or, for CALIB_FIX_ASPECT_RATIO, the aspect ratio K[0,0] / K[1,1]; D has at most
    5 coefficients.  criteria = (type, max_iter, epsilon) as cv2.TermCriteria.  Returns what cv2 returns, in its order: rms,
    K [3, 3], D [1, 5], rvecs and tvecs (tuples of [3, 1]), stdDeviationsIntrinsics [18, 1], stdDeviationsExtrinsics [6 n, 1] and
    perViewErrors [n, 1].  stats: an optional _lib.fid_calib_stats to fill."""
    return _run("fid_calibrate_camera", object_points, image_points, image_size, K, D, flags, criteria, device, stats)


def calibrate_camera_ro(object_points, image_points, image_size, fixed_point, K=None, D=None, flags=0, criteria=None, device=0, stats=None):
    """cv2.calibrateCameraROExtended(object_points, image_points, image_size, fixed_point, K, D, flags=flags, criteria=criteria) on
    the GPU: calibrate_camera that also re-estimates the board's points (the object-releasing method), for printed boards whose
    geometry is not exact.

    The points are released when 1 <= fixed_point <= n - 2 (n = the points of view 0); every view must then hold the same object
    points (charuco_views(..., complete=True) gives such views).  Point 0, point fixed_point and z of point n - 1 stay fixed.
    Returns cv2's 10-tuple in its order: rms, K, D, rvecs, tvecs, newObjPoints [1, n, 3] float32, stdDeviationsIntrinsics [18, 1],
    stdDeviationsExtrinsics [6 views, 1], stdDeviationsObjPoints [3 n, 1] and perViewErrors [views, 1]; with fixed_point out of
    range nothing is released, the result is calibrate_camera's and newObjPoints, stdDeviationsObjPoints are None, as in cv2."""
    n = len(np.asarray(object_points[0]).reshape(-1, 3)) if len(object_points) else 0
    new_obj, std_obj, rel = np.zeros((max(n, 1), 3), np.float32), np.zeros((max(n, 1), 3)), C.c_int(0)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    r = _run("fid_calibrate_camera_ro", object_points, image_points, image_size, K, D, flags, criteria, device, stats,
             (int(fixed_point), vp(new_obj), vp(std_obj), C.byref(rel)))
    rms, Kout, Dout, rv, tv, std_int, std_ext, pve = r
    if not rel.value:
        return rms, Kout, Dout, rv, tv, None, std_int, std_ext, None, pve
    return rms, Kout, Dout, rv, tv, new_obj[:n].reshape(1, n, 3).copy(), std_int, std_ext, std_obj[:n].reshape(-1, 1).copy(), pve


def charuco_views(board, corner_ids, corner_xy, complete=False):
    """Per frame ChArUco corners (the corner ids and corners of Detector.charuco / last_charuco for one board, one entry per frame)
    as calibration views, as cv2.aruco.CharucoBoard.matchImagePoints pairs them: object points [n][3] = the board's chessboard
    corners of the ids, image points [n][2], in detection order.  Frames with fewer than 4 corners, or whose corners are collinear
    on the board (cv2.calibrateCamera raises on them), are dropped.  With complete=True only frames in which every chessboard
    corner was found are kept, their corners in ascending id order: every view then holds the same object points, as
    calibrate_camera_ro needs to release them.  Returns (object_points, image_points, frame indices kept)."""
    sx = board.size[0] - 1
    obj, img, kept = [], [], []
    for f, (ids, xy) in enumerate(zip(corner_ids, corner_xy)):
        ids = np.asarray(ids, np.int64).reshape(-1)
        xy = np.asarray(xy, np.float32).reshape(-1, 2)
        if len(ids) < 4 or len(ids) != len(xy) or ids.min() < 0 or ids.max() >= board.n_corners:
            continue
        if complete:
            order = np.argsort(ids, kind="stable")
            ids, xy = ids[order], xy[order]
            if len(ids) != board.n_corners or np.any(ids != np.arange(board.n_corners)):
                continue
        g = np.stack([ids % sx, ids // sx], 1)  # board grid coordinates: collinearity is exact in integers
        d = g[1:] - g[0]
        if not np.any(d[:, 0, None] * d[None, :, 1] - d[:, 1, None] * d[None, :, 0]):
            continue
        obj.append(board.chessboard_corners[ids].copy())
        img.append(xy.copy())
        kept.append(f)
    return obj, img, kept
