"""cv2 oracle for the planar pose hypotheses of a square marker (fid_pose_hypotheses), and the seeded corner sets the tests feed
it.  TEST INFRASTRUCTURE ONLY.

``pose_hypotheses`` is ``cv2.solvePnPGeneric(obj, corners, K, D, flags=SOLVEPNP_IPPE_SQUARE)`` with the reference's float32 object
points (aruco_detect.cpp:151-161, ``aruco_oracle.single_marker_object_points``).  cv2 does not return the errors its IPPE solver
orders the two solutions by, so they are restated here (``IPPE::PoseSolver::evalReprojError``: projectPoints with K = I and no
distortion against the float32 output of cv::undistortPoints, summed in float32).  The basin of ``cv2.solvePnP`` (ITERATIVE, the
published pose) is the index of the solution whose rotation is closer to it.
"""
from __future__ import annotations

import math

import cv2
import numpy as np

from oracle import aruco_oracle as ao


def _closer(rvec_iter, rvecs) -> int:
    """Index of the rotation closest to rvec_iter (largest trace of R_i^T R_iter)."""
    Rit, _ = cv2.Rodrigues(np.asarray(rvec_iter, np.float64).reshape(3, 1))
    tr = [float(np.sum(cv2.Rodrigues(np.asarray(r, np.float64).reshape(3, 1))[0] * Rit)) for r in rvecs]
    return 1 if tr[1] > tr[0] else 0


def solver_errors(obj, corners, K, D, rvecs, tvecs):
    """IPPE::PoseSolver::evalReprojError of each solution (float32, normalised coordinates)."""
    un = cv2.undistortPoints(np.asarray(corners, np.float32).reshape(-1, 1, 2), K, D).reshape(-1, 2)  # float32, like cv2's
    out = []
    for rv, tv in zip(rvecs, tvecs):
        proj, _ = cv2.projectPoints(obj, rv, tv, np.eye(3), None)
        d = proj.reshape(-1, 2).astype(np.float32) - un.astype(np.float32)
        e = np.float32(0)
        for dx, dy in d:
            e = np.float32(e + np.float32(dx * dx) + np.float32(dy * dy))
        out.append(float(np.float32(math.sqrt(float(np.float32(e / np.float32(8.0)))))))
    return out


def pose_hypotheses(corners, K, D, marker_len):
    """Both IPPE_SQUARE solutions of one marker (corners float32 [4,2], TL TR BR BL) as solvePnPGeneric orders them.

    Returns dict(n, rvec [2,3], tvec [2,3], rms [2], solver_err [2], iterative_rvec [3], iterative_match)."""
    K = np.asarray(K, np.float64).reshape(3, 3)
    D = np.asarray(D, np.float64).reshape(-1)
    obj = ao.single_marker_object_points(float(marker_len))
    c = np.asarray(corners, np.float32).reshape(4, 2)
    n, rvecs, tvecs, rms = cv2.solvePnPGeneric(obj, c, K, D, flags=cv2.SOLVEPNP_IPPE_SQUARE)
    if n == 0:  # (cv2.solvePnP itself raises on such a quad)
        return dict(n=0, rvec=np.zeros((2, 3)), tvec=np.zeros((2, 3)), rms=np.zeros(2), solver_err=[0.0, 0.0], iterative_rvec=np.zeros(3), iterative_match=-1)
    _, rv_it, _ = cv2.solvePnP(obj, c, K, D)
    out = dict(n=int(n), iterative_rvec=rv_it.reshape(3))
    rvecs = np.array([r.reshape(3) for r in rvecs])
    tvecs = np.array([t.reshape(3) for t in tvecs])
    out.update(rvec=rvecs, tvec=tvecs, rms=np.asarray(rms, np.float64).reshape(2), solver_err=solver_errors(obj, c, K, D, rvecs, tvecs),
               iterative_match=_closer(rv_it, rvecs))
    return out


TOL = 1e-6


def assert_matches(got, ref, what=""):
    """The record against the oracle: rvec/tvec <= 1e-6, rms <= 1e-6 relative, identical order -- unless cv2's two ordering errors
    are within 1e-6 relative of each other, where the solutions may come swapped."""
    assert got["n"] == ref["n"], what
    if ref["n"] == 0:
        return False
    e0, e1 = ref["solver_err"]
    order = [0, 1]
    if not np.allclose(got["rvec"], ref["rvec"], rtol=0, atol=TOL) or not np.allclose(got["tvec"], ref["tvec"], rtol=0, atol=TOL):
        assert abs(e0 - e1) <= 1e-6 * max(e0, e1), (what, got, ref)  # a tie: the swap is accepted
        order = [1, 0]
    rv, tv, rms = ref["rvec"][order], ref["tvec"][order], ref["rms"][order]
    assert np.abs(got["rvec"] - rv).max() <= TOL, (what, got["rvec"], rv)
    assert np.abs(got["tvec"] - tv).max() <= TOL, (what, got["tvec"], tv)
    assert np.all(np.abs(got["rms"] - rms) <= TOL * np.maximum(rms, 1e-12)), (what, got["rms"], rms)
    assert got["iterative_match"] == order[ref["iterative_match"]], what
    return order == [1, 0]


def record_dict(r):
    """A fid_pose_hypotheses ctypes record as the dicts above."""
    return dict(n=int(r.n), iterative_match=int(r.iterative_match), rvec=np.array([list(v) for v in r.rvec]), tvec=np.array([list(v) for v in r.tvec]),
                rms=np.array(list(r.rms)))


def iterative_in_second_basin(K, D, seeds=range(200, 400)):
    """A seeded marker for which cv2.solvePnP (ITERATIVE) converges to the worse of the two IPPE solutions: (corners, len, ref)."""
    for seed in seeds:
        for c, L in synthetic_cases(seed, K, D, kind="far", n=20):
            ref = pose_hypotheses(c, K, D, L)
            if ref["n"] == 2 and ref["iterative_match"] == 1:
                return c, L, ref
    raise AssertionError("no case found")


# ---- seeded corner sets ------------------------------------------------------------------------------------------------------
def _rot(axis_angle):
    R, _ = cv2.Rodrigues(np.asarray(axis_angle, np.float64).reshape(3, 1))
    return R


def marker_corners(R, t, K, D, marker_len, rng=None, noise=0.0):
    """float32 corners [4,2] of a marker at pose (R, t), projected with K and D (+ optional pixel noise)."""
    obj = ao.single_marker_object_points(marker_len).astype(np.float64)
    rv, _ = cv2.Rodrigues(R)
    img, _ = cv2.projectPoints(obj, rv, np.asarray(t, np.float64), K, D)
    img = img.reshape(4, 2)
    if noise:
        img = img + rng.normal(0.0, noise, img.shape)
    return img.astype(np.float32)


def synthetic_cases(seed, K, D, W=640, H=480, n=40, kind="mixed"):
    """Seeded (corners, marker_len) sets.  kinds: "far" = small, distant, nearly fronto-parallel markers (the two solutions come
    close), "tilted" = 55-80 degrees out of plane, "mixed" = anything in between."""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n:
        L = float(rng.choice([0.05, 0.1, 0.14, 0.2]))
        if kind == "far":
            tilt, z = rng.uniform(0.0, 0.2), rng.uniform(2.5, 7.0)
        elif kind == "tilted":
            tilt, z = rng.uniform(0.95, 1.4), rng.uniform(0.4, 2.0)
        else:
            tilt, z = rng.uniform(0.0, 1.2), rng.uniform(0.3, 4.0)
        ax = rng.normal(size=3)
        ax[2] = 0.0
        ax /= np.linalg.norm(ax)
        # marker facing the camera (x right, y up in the marker -> image y down), tilted about an in-plane axis, spun in-plane
        R = _rot([math.pi, 0.0, 0.0]) @ _rot(ax * tilt) @ _rot([0.0, 0.0, rng.uniform(-math.pi, math.pi)])
        u, v = rng.uniform(0.15 * W, 0.85 * W), rng.uniform(0.15 * H, 0.85 * H)
        t = z * np.array([(u - K[0, 2]) / K[0, 0], (v - K[1, 2]) / K[1, 1], 1.0])
        c = marker_corners(R, t, K, D, L, rng, noise=float(rng.uniform(0.0, 0.3)))
        if c.min() < 0 or c[:, 0].max() > W - 1 or c[:, 1].max() > H - 1:
            continue
        if cv2.contourArea(c) < 64.0:
            continue
        out.append((c, L))
    return out
