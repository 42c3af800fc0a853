"""cv2 oracle for the ChArUco diamonds (fid_detect_diamonds, fid_last_diamonds), and the rendered diamond frames the tests feed it.
TEST INFRASTRUCTURE ONLY.

``detect`` is what a cv2 user computes with markers already detected: ``cv2.aruco.CharucoDetector(CharucoBoard((3, 3),
squareLength, markerLength, dict), params, detector_params).detectDiamonds(image, markerCorners=..., markerIds=...)`` with the
project's detector parameters.  ``pose`` continues with ``cv2.solvePnP(SOLVEPNP_ITERATIVE)`` of each diamond's four corners on
``getSingleMarkerObjectPoints(squareLength)``, the published FiducialTransform arithmetic on top.
"""
from __future__ import annotations

import math

import cv2
import numpy as np

import charuco_oracle as co
from oracle import aruco_oracle as ao

DICT = co.DICT
DICT_ID = co.DICT_ID


def detector(square, marker, K=None, D=None, min_markers=2, check_markers=True, method=cv2.aruco.CORNER_REFINE_SUBPIX):
    cp = cv2.aruco.CharucoParameters()
    if K is not None:
        cp.cameraMatrix = np.asarray(K, np.float64).reshape(3, 3)
        cp.distCoeffs = np.asarray(D, np.float64).reshape(1, -1)
    cp.minMarkers = int(min_markers)
    cp.checkMarkers = bool(check_markers)
    dp = ao.reference_detector_params(cornerRefinementMethod=method)
    return cv2.aruco.CharucoDetector(cv2.aruco.CharucoBoard((3, 3), square, marker, DICT), cp, dp)


def detect_markers(gray, method=cv2.aruco.CORNER_REFINE_SUBPIX):
    """detectMarkers with the project's detector parameters: ids [n] int32, corners [n, 4, 2] float32."""
    det = cv2.aruco.ArucoDetector(DICT, ao.reference_detector_params(cornerRefinementMethod=method))
    corners, ids, _ = det.detectMarkers(gray)
    ids = np.zeros(0, np.int32) if ids is None else ids.reshape(-1).astype(np.int32)
    return ids, np.array(corners, np.float32).reshape(-1, 4, 2)


def detect(det, gray, ids, corners, markers_after=False):
    """detectDiamonds with the given markers: (ids [k, 4] int32, corners [k, 4, 2] float32), in cv2's order.  markers_after: also
    the marker corners [n, 4, 2] cv2 hands back -- under CORNER_REFINE_SUBPIX it writes the cornerSubPix of every marker it recovers
    into them (DESIGN.md finding 13)."""
    ids = np.asarray(ids, np.int32).reshape(-1, 1)
    cs = tuple(np.asarray(c, np.float32).reshape(1, 4, 2).copy() for c in np.asarray(corners, np.float32).reshape(-1, 4, 2))
    dc, di, mc, _ = det.detectDiamonds(gray, markerCorners=cs, markerIds=ids)
    mc = np.array(mc, np.float32).reshape(-1, 4, 2)
    if di is None or len(di) == 0:
        out = np.zeros((0, 4), np.int32), np.zeros((0, 4, 2), np.float32)
    else:
        out = np.asarray(di).reshape(-1, 4).astype(np.int32), np.array(dc, np.float32).reshape(-1, 4, 2)
    return out + (mc,) if markers_after else out


def pose(corners, square, K, D):
    """solvePnP(ITERATIVE) of one diamond on getSingleMarkerObjectPoints(square): dict(rvec, tvec, rotation (x y z w), image_error)."""
    h = np.float32(square) / np.float32(2)
    obj = np.array([[-h, h, 0], [h, h, 0], [h, -h, 0], [-h, -h, 0]], np.float32)
    img = np.asarray(corners, np.float32).reshape(4, 2)
    K = np.asarray(K, np.float64).reshape(3, 3)
    D = np.asarray(D, np.float64).reshape(-1)
    ok, rv, tv = cv2.solvePnP(obj, img, K, D, flags=cv2.SOLVEPNP_ITERATIVE)
    assert ok
    rv, tv = rv.reshape(3), tv.reshape(3)
    proj, _ = cv2.projectPoints(obj, rv, tv, K, D)
    d = np.hypot(*(img.astype(np.float64) - proj.reshape(-1, 2)).T)
    angle = float(np.linalg.norm(rv))
    q = np.concatenate([rv / angle * math.sin(angle / 2), [math.cos(angle / 2)]])
    return dict(rvec=rv, tvec=tv, rotation=q, image_error=float(np.sum(d * d) / 4))


# ---- rendered diamonds ----------------------------------------------------------------------------------------------------------
def _rot(v):
    return cv2.Rodrigues(np.asarray(v, np.float64).reshape(3, 1))[0]


def diamond_pose(rng, K, W, H, square, kind, centre, spin):
    """A pose (R, t) of a 3x3 diamond with its centre at image point `centre`: near, far or oblique, turned in its plane by spin
    quarter turns (plus a little)."""
    c = np.array([1.5 * square, 1.5 * square, 0.0])
    ext = 3 * square
    f = K[0, 0]
    frac = {"near": (0.3, 0.45), "far": (0.12, 0.18), "oblique": (0.25, 0.35)}[kind]
    tilt = rng.uniform(0.6, 0.9) if kind == "oblique" else rng.uniform(0.0, 0.35)
    z = ext * f / rng.uniform(*frac) / W
    ax = rng.normal(size=3)
    ax[2] = 0.0
    ax /= np.linalg.norm(ax)
    R = _rot(ax * tilt) @ _rot([0.0, 0.0, spin * math.pi / 2 + rng.uniform(-0.3, 0.3)])
    u, v = centre
    t = z * np.array([(u - K[0, 2]) / K[0, 0], (v - K[1, 2]) / K[1, 1], 1.0]) - R @ c
    return R, t


def render_diamond(gray, ids, square, marker, R, t, K):
    co.render(gray, cv2.aruco.CharucoBoard((3, 3), square, marker, DICT, np.asarray(ids, np.int32)), R, t, K)


def cover_marker(gray, square, marker, k, R, t, K):
    """Paint over marker k (board order) of a rendered diamond, a little beyond its outline."""
    b = cv2.aruco.CharucoBoard((3, 3), square, marker, DICT)
    o = np.asarray(b.getObjPoints()[k], np.float64).reshape(4, 3)
    c = o.mean(axis=0)
    o = c + (o - c) * 1.15
    p = co.project(o, R, t, K, np.zeros(5))
    cv2.fillConvexPoly(gray, np.round(p).astype(np.int32), 255)


def render_stray(gray, mid, length, R, t, K):
    """A single marker of side `length` at pose (R, t) (its top-left corner at the origin), in place."""
    px = 60
    img = cv2.aruco.generateImageMarker(DICT, int(mid), px)
    img = cv2.copyMakeBorder(img, px // 6, px // 6, px // 6, px // 6, cv2.BORDER_CONSTANT, value=255)
    s = length / px
    m = px // 6
    A = np.array([[s, 0, -m * s], [0, s, -m * s], [0, 0, 1]])
    Hm = np.asarray(K, np.float64) @ np.column_stack([R[:, 0], R[:, 1], t]) @ A
    H, W = gray.shape
    warped = cv2.warpPerspective(img, Hm, (W, H), flags=cv2.INTER_LINEAR)
    mask = cv2.warpPerspective(np.full_like(img, 255), Hm, (W, H), flags=cv2.INTER_NEAREST)
    gray[mask > 0] = warped[mask > 0]
