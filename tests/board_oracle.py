"""cv2 oracle for one pose per marker board (fid_estimate_board_poses, fid_last_board_poses), and the seeded boards and detection
lists the tests feed it.  TEST INFRASTRUCTURE ONLY.

``board_pose`` is what a cv2 user computes: ``cv2.aruco.Board(obj, dictionary, ids).matchImagePoints(corners, ids)`` and then
``cv2.solvePnP(obj, img, K, D, flags=SOLVEPNP_ITERATIVE)``; status -1 where solvePnP raises, 0 where no board marker was
detected.  ``image_error`` is getReprojectionError (aruco_detect.cpp:203-221) over every matched point: the mean of the squared
distances to ``cv2.projectPoints``'s projections rounded to float32.
"""
from __future__ import annotations

import math

import cv2
import numpy as np

from fiducials_b200.board import Board, grid_board

DICT = cv2.aruco.getPredefinedDictionary(cv2.aruco.DICT_6X6_250)


def cv_board(board: Board):
    return cv2.aruco.Board([np.ascontiguousarray(o, np.float32) for o in board.obj_points], DICT, board.ids.reshape(-1, 1))


def match(board: Board, ids, corners):
    """Board.matchImagePoints on a detection list: (obj [N,3] float32, img [N,2] float32)."""
    ids = np.asarray(ids, np.int32).reshape(-1)
    if len(ids) == 0:
        return np.zeros((0, 3), np.float32), np.zeros((0, 2), np.float32)
    cs = [np.asarray(c, np.float32).reshape(1, 4, 2) for c in np.asarray(corners, np.float32).reshape(-1, 4, 2)]
    obj, img = cv_board(board).matchImagePoints(cs, ids.reshape(-1, 1))
    if obj is None or len(obj) == 0:
        return np.zeros((0, 3), np.float32), np.zeros((0, 2), np.float32)
    return obj.reshape(-1, 3).astype(np.float32), img.reshape(-1, 2).astype(np.float32)


def board_pose(board: Board, ids, corners, K, D):
    """dict(status, n_markers, n_points, rvec, tvec, rotation (quaternion x y z w), image_error) as a cv2 user gets them."""
    K = np.asarray(K, np.float64).reshape(3, 3)
    D = np.asarray(D, np.float64).reshape(-1)
    obj, img = match(board, ids, corners)
    out = dict(status=0, n_markers=len(obj) // 4, n_points=len(obj), rvec=np.zeros(3), tvec=np.zeros(3), rotation=np.zeros(4), image_error=0.0)
    if len(obj) == 0:
        return out
    try:
        ok, rv, tv = cv2.solvePnP(obj, img, K, D, flags=cv2.SOLVEPNP_ITERATIVE)
    except cv2.error:
        out["status"] = -1
        return out
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


TOL = 1e-6


def assert_matches(got, ref, what="", tol=TOL):
    """status, counts identical; rvec / tvec within tol absolute, image_error within tol relative.  Returns the differences."""
    assert got["status"] == ref["status"], (what, got["status"], ref["status"])
    assert got["n_markers"] == ref["n_markers"] and got["n_points"] == ref["n_points"], (what, got, ref)
    if ref["status"] != 1:
        return 0.0, 0.0
    dp = max(np.abs(np.asarray(got["rvec"]) - ref["rvec"]).max(), np.abs(np.asarray(got["tvec"]) - ref["tvec"]).max())
    de = abs(got["image_error"] - ref["image_error"]) / max(ref["image_error"], 1e-300)
    assert dp <= tol, (what, got["rvec"], got["tvec"], ref["rvec"], ref["tvec"])
    assert de <= tol or abs(got["image_error"] - ref["image_error"]) <= 1e-12, (what, got["image_error"], ref["image_error"])
    assert np.abs(np.asarray(got["rotation"]) - ref["rotation"]).max() <= 10 * tol, what
    return dp, de


def record_dict(r):
    """A fid_board_pose ctypes record as the dicts above."""
    return dict(board=int(r.board), status=int(r.status), n_markers=int(r.n_markers), n_points=int(r.n_points), rvec=np.array(list(r.rvec)),
                tvec=np.array(list(r.tvec)), rotation=np.array(list(r.rotation)), image_error=float(r.image_error))


# ---- seeded boards and detection lists ---------------------------------------------------------------------------------------
def _rot(v):
    return cv2.Rodrigues(np.asarray(v, np.float64).reshape(3, 1))[0]


def project(obj, R, t, K, D, rng=None, noise=0.0):
    rv, _ = cv2.Rodrigues(R)
    img, _ = cv2.projectPoints(np.asarray(obj, np.float64).reshape(-1, 3), rv, np.asarray(t, np.float64), K, D)
    img = img.reshape(-1, 2)
    if noise:
        img = img + rng.normal(0.0, noise, img.shape)
    return img.astype(np.float32)


def board_in_view(board, rng, K, W=640, H=480, kind="near"):
    """A pose (R, t) that puts the board's centre in front of the camera: near, far or oblique."""
    c = board.obj_points.reshape(-1, 3).astype(np.float64).mean(0)
    ext = float(np.ptp(board.obj_points.reshape(-1, 3), axis=0).max())
    f = K[0, 0]
    if kind == "near":
        tilt, z = rng.uniform(0.0, 0.5), ext * f / rng.uniform(0.5, 0.8) / W
    elif kind == "far":
        tilt, z = rng.uniform(0.0, 0.3), ext * f / rng.uniform(0.12, 0.25) / W
    else:  # oblique
        tilt, z = rng.uniform(0.8, 1.15), ext * f / rng.uniform(0.4, 0.7) / W
    ax = rng.normal(size=3)
    ax[2] = 0.0
    ax /= np.linalg.norm(ax)
    R = _rot([math.pi, 0.0, 0.0]) @ _rot(ax * tilt) @ _rot([0.0, 0.0, rng.uniform(-0.6, 0.6)])
    u, v = rng.uniform(0.4 * W, 0.6 * W), rng.uniform(0.4 * H, 0.6 * H)
    t = z * np.array([(u - K[0, 2]) / K[0, 0], (v - K[1, 2]) / K[1, 1], 1.0]) - R @ c
    return R, t


def detections(board, R, t, K, D, rng, noise=0.0, keep=None, extra_ids=(), repeat=0, shuffle=True):
    """A detection list (ids [n], corners [n,4,2] float32) of the board at pose (R, t): the markers `keep` (default all), in
    shuffled order, plus markers whose ids are off the board and `repeat` repeated detections."""
    idx = list(range(len(board))) if keep is None else list(keep)
    ids = [int(board.ids[k]) for k in idx]
    cs = [project(board.obj_points[k], R, t, K, D, rng, noise).reshape(4, 2) for k in idx]
    for j in range(repeat):
        k = int(rng.integers(len(idx)))
        ids.append(ids[k])
        cs.append(cs[k] + rng.normal(0.0, 0.2, (4, 2)).astype(np.float32))
    for e in extra_ids:
        ids.append(int(e))
        cs.append(rng.uniform(0, 400, (4, 2)).astype(np.float32))
    order = rng.permutation(len(ids)) if shuffle else np.arange(len(ids))
    return np.array([ids[o] for o in order], np.int32), np.array([cs[o] for o in order], np.float32).reshape(-1, 4, 2)


def transformed(board, R, t):
    """The board moved rigidly (float32 points): a plane that is no longer z = 0."""
    obj = (board.obj_points.reshape(-1, 3).astype(np.float64) @ np.asarray(R).T + np.asarray(t)).astype(np.float32)
    return Board(board.ids, obj.reshape(-1, 4, 3))


def cube_board(n_faces, side=0.2, marker=0.12, first_id=0):
    """Markers on n_faces (2 or 3) faces of a cube, one per face, each seen from outside: a non-planar board."""
    h, m = side / 2, marker / 2
    sq = np.array([[-m, m], [m, m], [m, -m], [-m, -m]])
    faces = [  # (origin of the face, its in-plane x and y axes)
        (np.array([0, 0, -h]), np.array([1, 0, 0]), np.array([0, -1, 0])),
        (np.array([h, 0, 0]), np.array([0, 0, 1]), np.array([0, -1, 0])),
        (np.array([0, -h, 0]), np.array([1, 0, 0]), np.array([0, 0, 1])),
    ]
    obj = [np.array([o + a * ex + b * ey for a, b in sq]) for o, ex, ey in faces[:n_faces]]
    return Board(np.arange(first_id, first_id + n_faces), np.array(obj, np.float32))


def bent_marker(marker=0.1, bend=0.02):
    """One marker whose 4 corners are not coplanar (one corner lifted): non-planar with 4 points, where cv2.solvePnP raises."""
    m = marker / 2
    return Board([5], np.array([[[-m, m, 0], [m, m, 0], [m, -m, bend], [-m, -m, 0]]], np.float32))


def grid_cases(seed, K, D, n=12):
    """Seeded (board, ids, corners): GridBoards 2x2 .. 10x10 at near, far and oblique poses, visible subsets down to one marker,
    0 - 0.5 px corner noise, ids off the board and repeated detections."""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n:
        w, h = int(rng.integers(2, 11)), int(rng.integers(2, 11))
        L = float(rng.choice([0.02, 0.04, 0.05, 0.1]))
        sep = float(L * rng.choice([0.1, 0.2, 0.25, 0.5]))
        ids = None if rng.random() < 0.5 else rng.permutation(250)[: w * h]
        b = grid_board((w, h), L, sep, ids)
        R, t = board_in_view(b, rng, K, kind=["near", "far", "oblique"][len(out) % 3])
        n_keep = int(rng.integers(1, len(b) + 1)) if rng.random() < 0.6 else len(b)
        keep = sorted(rng.choice(len(b), n_keep, replace=False).tolist())
        extra = [int(e) for e in rng.integers(250, 1000, int(rng.integers(0, 3)))]
        di, dc = detections(b, R, t, K, D, rng, noise=float(rng.uniform(0.0, 0.5)), keep=keep, extra_ids=extra, repeat=int(rng.random() < 0.2))
        if np.abs(dc).max() > 5000:
            continue
        out.append((b, di, dc))
    return out
