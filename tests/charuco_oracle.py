"""cv2 oracle for the ChArUco corners and pose (fid_detect_charuco, fid_last_charuco), and the rendered ChArUco frames the tests feed
it.  TEST INFRASTRUCTURE ONLY.

``detect`` is what a cv2 user computes with markers already detected: ``cv2.aruco.CharucoDetector(board, params, detector_params)
.detectBoard(image, markerCorners=..., markerIds=...)``.  ``pose`` continues with ``board.matchImagePoints(corners, ids)`` and
``cv2.solvePnP(SOLVEPNP_ITERATIVE)`` where a cv2 user may call it: a camera, at least 4 corners and
``board.checkCharucoCornersCollinear(ids)`` false.
"""
from __future__ import annotations

import math

import cv2
import numpy as np

DICT = cv2.aruco.getPredefinedDictionary(cv2.aruco.DICT_6X6_250)
DICT_ID = 10  # DICT_6X6_250 in fid_params.dictionary
# the detector parameters of fiducials_b200.node.default_params that detectBoard reads
REFINE_WIN, REFINE_MAX_ITER, REFINE_MIN_ACC = 5, 30, 0.01


def cv_board(size, square, marker, ids=None, legacy=False):
    b = cv2.aruco.CharucoBoard(tuple(size), square, marker, DICT, None if ids is None else np.asarray(ids, np.int32))
    b.setLegacyPattern(bool(legacy))
    return b


def detect(board, image, ids, corners, K=None, D=None, min_markers=2, check_markers=True):
    """detectBoard with the given markers: (corner ids [n] int32, corners [n,2] float32)."""
    cp = cv2.aruco.CharucoParameters()
    if K is not None:
        cp.cameraMatrix = np.asarray(K, np.float64).reshape(3, 3)
        cp.distCoeffs = np.asarray(D, np.float64).reshape(1, -1)
    cp.minMarkers = int(min_markers)
    cp.checkMarkers = bool(check_markers)
    dp = cv2.aruco.DetectorParameters()
    dp.cornerRefinementWinSize = REFINE_WIN
    dp.cornerRefinementMaxIterations = REFINE_MAX_ITER
    dp.cornerRefinementMinAccuracy = REFINE_MIN_ACC
    det = cv2.aruco.CharucoDetector(board, cp, dp)
    ids = np.asarray(ids, np.int32).reshape(-1, 1)
    cs = tuple(np.asarray(c, np.float32).reshape(1, 4, 2) for c in np.asarray(corners, np.float32).reshape(-1, 4, 2))
    ch_corners, ch_ids, _, _ = det.detectBoard(image, markerCorners=cs, markerIds=ids)
    if ch_ids is None or len(ch_ids) == 0:
        return np.zeros(0, np.int32), np.zeros((0, 2), np.float32)
    return ch_ids.reshape(-1).astype(np.int32), ch_corners.reshape(-1, 2).astype(np.float32)


def pose(board, ch_ids, ch_corners, K, D, rejected=False):
    """dict(status, rvec, tvec, rotation (quaternion x y z w), image_error) for the corners detect returned: status 1 pose, 0 no
    camera or fewer than 4 corners, -2 collinear corners, -3 (given as `rejected`) the board check dropped every corner."""
    out = dict(status=0, rvec=np.zeros(3), tvec=np.zeros(3), rotation=np.zeros(4), image_error=0.0)
    if rejected:
        out["status"] = -3
        return out
    if K is None or len(ch_ids) < 4:
        return out
    if board.checkCharucoCornersCollinear(np.asarray(ch_ids, np.int32).reshape(-1, 1)):
        out["status"] = -2
        return out
    K = np.asarray(K, np.float64).reshape(3, 3)
    D = np.asarray(D, np.float64).reshape(-1)
    obj, img = board.matchImagePoints(np.asarray(ch_corners, np.float32).reshape(-1, 1, 2), np.asarray(ch_ids, np.int32).reshape(-1, 1))
    obj, img = obj.reshape(-1, 3).astype(np.float32), img.reshape(-1, 2).astype(np.float32)
    ok, rv, tv = cv2.solvePnP(obj, img, K, D, flags=cv2.SOLVEPNP_ITERATIVE)
    assert ok
    rv, tv = rv.reshape(3), tv.reshape(3)
    proj, _ = cv2.projectPoints(obj, rv, tv, K, D)
    proj = proj.reshape(-1, 2).astype(np.float32).astype(np.float64)
    d = np.hypot(img[:, 0].astype(np.float64) - proj[:, 0], img[:, 1].astype(np.float64) - proj[:, 1])
    angle = float(np.linalg.norm(rv))
    ax = rv / angle
    q = np.concatenate([ax * math.sin(angle / 2) / np.linalg.norm(ax), [math.cos(angle / 2)]])
    out.update(status=1, rvec=rv, tvec=tv, rotation=q, image_error=float(np.sum(d * d) / len(d)))
    return out


def full(board, image, ids, corners, K=None, D=None, min_markers=2, check_markers=True):
    """detect + pose; the board check's rejection is told apart from an empty result by detecting once more without it."""
    ch_ids, ch_xy = detect(board, image, ids, corners, K, D, min_markers, check_markers)
    rejected = False
    if len(ch_ids) == 0 and check_markers:
        rejected = len(detect(board, image, ids, corners, K, D, min_markers, False)[0]) > 0
    return ch_ids, ch_xy, pose(board, ch_ids, ch_xy, K, D, rejected)


# measured: 1 135 of 1 140 corners bit-identical on the host, the others up to 1.3e-3 px off (cornerSubPix walks through a nearly
# flat window, where a last-bit difference moves the converged point; DESIGN.md finding 9)
CORNER_TOL = 2e-3
POSE_TOL = 1e-6


def assert_matches(got_ids, got_xy, got_pose, ref_ids, ref_xy, ref_pose, what=""):
    """ids identical and in order; corners within CORNER_TOL px; status identical; rvec / tvec within POSE_TOL, image_error within
    POSE_TOL relative.  Returns (max corner difference, max pose difference)."""
    assert np.array_equal(np.asarray(got_ids), np.asarray(ref_ids)), (what, got_ids, ref_ids)
    dc = float(np.abs(np.asarray(got_xy, np.float64) - ref_xy).max()) if len(ref_ids) else 0.0
    assert dc <= CORNER_TOL, (what, dc)
    assert got_pose["status"] == ref_pose["status"], (what, got_pose["status"], ref_pose["status"])
    if ref_pose["status"] != 1:
        return dc, 0.0
    dp = max(np.abs(np.asarray(got_pose["rvec"]) - ref_pose["rvec"]).max(), np.abs(np.asarray(got_pose["tvec"]) - ref_pose["tvec"]).max())
    assert dp <= POSE_TOL, (what, got_pose, ref_pose)
    de = abs(got_pose["image_error"] - ref_pose["image_error"])
    assert de <= POSE_TOL * ref_pose["image_error"] or de <= 1e-12, (what, got_pose["image_error"], ref_pose["image_error"])
    assert np.abs(np.asarray(got_pose["rotation"]) - ref_pose["rotation"]).max() <= 10 * POSE_TOL, what
    return dc, dp


# ---- rendered boards ------------------------------------------------------------------------------------------------------------
def _rot(v):
    return cv2.Rodrigues(np.asarray(v, np.float64).reshape(3, 1))[0]


def project(obj, R, t, K, D):
    rv, _ = cv2.Rodrigues(R)
    img, _ = cv2.projectPoints(np.asarray(obj, np.float64).reshape(-1, 3), rv, np.asarray(t, np.float64), K, D)
    return img.reshape(-1, 2)


def render(gray, board, R, t, K, px_per_square=60, margin=None):
    """CharucoBoard.generateImage of the board, warped into the gray frame at pose (R, t) through K (no distortion), in place."""
    sx, sy = board.getChessboardSize()
    sq = board.getSquareLength()
    margin = px_per_square // 2 if margin is None else margin
    bw, bh = sx * px_per_square + 2 * margin, sy * px_per_square + 2 * margin
    img = board.generateImage((bw, bh), marginSize=margin, borderBits=1)
    s = sq / px_per_square
    A = np.array([[s, 0, -margin * s], [0, s, -margin * s], [0, 0, 1]])  # image px -> board metres
    Hm = np.asarray(K, np.float64) @ np.column_stack([R[:, 0], R[:, 1], t]) @ A
    H, W = gray.shape
    warped = cv2.warpPerspective(img, Hm, (W, H), flags=cv2.INTER_LINEAR)
    mask = cv2.warpPerspective(np.full_like(img, 255), Hm, (W, H), flags=cv2.INTER_NEAREST)
    gray[mask > 0] = warped[mask > 0]


def board_pose_in_view(board, rng, K, W, H, kind="near", centre=None):
    """A pose (R, t) that puts the board's centre in front of the camera: near, far or oblique (x right, y down as printed)."""
    sx, sy = board.getChessboardSize()
    sq = board.getSquareLength()
    c = np.array([sx * sq / 2, sy * sq / 2, 0.0])
    ext = max(sx, sy) * sq
    f = K[0, 0]
    if kind == "near":
        tilt, z = rng.uniform(0.0, 0.4), ext * f / rng.uniform(0.5, 0.8) / W
    elif kind == "far":
        tilt, z = rng.uniform(0.0, 0.3), ext * f / rng.uniform(0.25, 0.4) / W
    else:  # oblique
        tilt, z = rng.uniform(0.6, 0.9), ext * f / rng.uniform(0.4, 0.7) / W
    ax = rng.normal(size=3)
    ax[2] = 0.0
    ax /= np.linalg.norm(ax)
    R = _rot(ax * tilt) @ _rot([0.0, 0.0, rng.uniform(-0.5, 0.5)])
    u, v = centre if centre is not None else (rng.uniform(0.4 * W, 0.6 * W), rng.uniform(0.4 * H, 0.6 * H))
    t = z * np.array([(u - K[0, 2]) / K[0, 0], (v - K[1, 2]) / K[1, 1], 1.0]) - R @ c
    return R, t


def marker_detections(board, R, t, K, D, rng, noise=0.0, keep=None, extra_ids=(), repeat=0, shuffle=True):
    """Marker detections (ids [n] int32, corners [n,4,2] float32) of the board at pose (R, t), projected through (K, D): the
    markers `keep` (default all), shuffled, `repeat` repeated detections and foreign ids."""
    obj = np.array(board.getObjPoints(), np.float64).reshape(-1, 4, 3)
    bids = np.asarray(board.getIds()).reshape(-1)
    idx = list(range(len(bids))) if keep is None else list(keep)
    ids = [int(bids[k]) for k in idx]
    cs = [project(obj[k], R, t, K, D) + (rng.normal(0.0, noise, (4, 2)) if noise else 0.0) for k in idx]
    for _ in range(repeat):
        k = int(rng.integers(len(idx)))
        ids.append(ids[k])
        cs.append(cs[k] + rng.normal(0.0, 0.2, (4, 2)))
    for e in extra_ids:
        ids.append(int(e))
        cs.append(rng.uniform(0, 400, (4, 2)))
    order = rng.permutation(len(ids)) if shuffle else np.arange(len(ids))
    return np.array([ids[o] for o in order], np.int32), np.array([cs[o] for o in order], np.float32).reshape(-1, 4, 2)


def blur_noise(gray, rng, blur=True, noise=0.0):
    out = cv2.GaussianBlur(gray, (5, 5), 1.0) if blur else gray.copy()
    if noise:
        out = np.clip(out.astype(np.float64) + rng.normal(0.0, noise * 255.0 / 8.0, out.shape), 0, 255).astype(np.uint8)
    return out
