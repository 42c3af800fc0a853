"""Seeded corner sets for the per-marker pose (solve_marker_pose: fid_pose, k_finish, k_recovered_pose) and its cv2 oracle.
TEST INFRASTRUCTURE ONLY.

``cases(cls, seed, n)`` draws ``n`` markers of one geometry class, each a marker projected with ``cv2.projectPoints`` (plus optional
pixel noise) and kept only when ``detectable`` -- the detector's own quad rules -- accepts it, since those are the only quads
``detectMarkers`` can hand to the pose.  ``oracle`` is what the reference node publishes for one marker: ``cv2.solvePnP`` (ITERATIVE)
on the reference's float32 object points, and the message fields of ``aruco_oracle.pose_fields`` / ``reprojection_error``.
``gauss_newton`` is an independent float64 minimiser of the same reprojection error, used to tell which of two disagreeing answers
is the better minimum.  Every case carries (class, seed, index) so that a failure names the case it came from.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import cv2
import numpy as np

from fiducials_b200 import synth
from oracle import aruco_oracle as ao
from ippe_oracle import _rot, marker_corners

FLEN = 0.14  # fiducial_len: the default marker length, not exact in float32
# per-id overrides (ids 1..): 0.05-1.0, some exact in float32 and some not
OVERRIDES = {1: 0.05, 2: 0.1, 3: 0.2, 4: 1.0 / 3.0, 5: 0.5, 6: 1.0, 7: 0.07}
LM_CAP = 20  # CvLevMarq's iteration limit in cvFindExtrinsicCameraParams2

_K640, _DREF = synth.camera_for(640, 480)
_DZERO = np.zeros(5)
_DSTRONG = np.array([-0.35, 0.12, 0.011, -0.009, -0.025])  # barrel, k3 != 0, p1 / p2 ~ 1e-2
_KANISO = np.array([[520.0, 0.0, 300.5], [0.0, 489.0, 255.25], [0.0, 0.0, 1.0]])
_K4K = np.array([[1400.0, 0.0, 1800.0], [0.0, 1330.0, 1150.0], [0.0, 0.0, 1.0]])

# class -> (K, D, W, H)
CAMERAS = {
    "mixed": (_K640, _DREF, 640, 480),
    "far": (_K640, _DREF, 640, 480),
    "grazing": (_K640, _DREF, 640, 480),
    "half_turn": (_K640, _DREF, 640, 480),
    "half_turn_d0": (_K640, _DZERO, 640, 480),
    "noisy": (_K640, _DREF, 640, 480),
    "strong_distortion": (_K640, _DSTRONG, 640, 480),
    "d_zero": (_K640, _DZERO, 640, 480),
    "aniso_640": (_KANISO, _DREF, 640, 480),
    "aniso_4k": (_K4K, _DREF, 3840, 2160),
}
CLASSES = tuple(CAMERAS)


@dataclass
class Case:
    cls: str
    seed: int
    index: int
    corners: np.ndarray  # float32 [4,2], TL TR BR BL
    marker_id: int  # 0 = the default length, else a key of OVERRIDES
    length: float  # the marker's side as the pose sees it: narrowed to float32

    @property
    def name(self):
        return "%s seed %d #%d" % (self.cls, self.seed, self.index)


def detectable(quad, W, H) -> bool:
    """The detector's quad rules (default DetectorParameters): convex; perimeter within [0.1, 4] x max(W, H); every side at least
    0.05 x perimeter; every corner at least minDistanceToBorder = 3 px inside the frame."""
    q = np.asarray(quad, np.float64).reshape(4, 2)
    if not np.all(np.isfinite(q)):
        return False
    sides = np.linalg.norm(q - np.roll(q, -1, axis=0), axis=1)
    per = float(sides.sum())
    mx = max(W, H)
    if not (0.1 * mx <= per <= 4.0 * mx) or sides.min() < 0.05 * per:
        return False
    if not cv2.isContourConvex(q.astype(np.float32).reshape(-1, 1, 2)):
        return False
    return q.min() >= 3 and q[:, 0].max() <= W - 4 and q[:, 1].max() <= H - 4


def _pose(rng, cls, W, H, L):
    """(R, centre pixel, depth / L, noise px) of one draw of the class."""
    ax = rng.normal(size=3)
    ax[2] = 0.0
    ax /= np.linalg.norm(ax)
    u, v = rng.uniform(0.1 * W, 0.9 * W), rng.uniform(0.1 * H, 0.9 * H)
    spin = rng.uniform(-math.pi, math.pi)
    if cls in ("mixed", "d_zero", "aniso_640", "aniso_4k"):
        tilt, zl, noise = rng.uniform(0.0, 1.2), rng.uniform(2.0, 30.0), rng.uniform(0.0, 0.3)
    elif cls == "far":  # down to the detector's minimum perimeter
        tilt, zl, noise = rng.uniform(0.0, 0.25), rng.uniform(14.0, 32.0), rng.uniform(0.0, 0.3)
    elif cls == "grazing":  # 70-88 degrees out of plane
        tilt, zl, noise = rng.uniform(math.radians(70), math.radians(88)), rng.uniform(1.5, 8.0), rng.uniform(0.0, 0.1)
    elif cls.startswith("half_turn"):  # squarely facing the camera, spin 0 / pi/2 / pi / -pi/2, or 1e-7..1e-3 rad off them
        off = [0.0, 1e-7, -1e-7, 1e-6, 1e-5, -1e-5, 1e-4, 1e-3]
        tilt = float(rng.choice([0.0, 0.0, 1e-7, 1e-6, 1e-5, 1e-3]))
        spin = float(rng.choice([0.0, math.pi / 2, math.pi, -math.pi / 2])) + float(rng.choice(off))
        zl, noise = rng.uniform(2.0, 20.0), 0.0
        if rng.uniform() < 0.2:  # centred on the principal point as well
            u, v = 0.5 * W, 0.5 * H
    elif cls == "noisy":
        tilt, zl, noise = rng.uniform(0.0, 1.2), rng.uniform(3.0, 25.0), rng.uniform(0.5, 1.5)
    elif cls == "strong_distortion":  # markers in the frame corners
        u = float(rng.choice([rng.uniform(0.04, 0.2), rng.uniform(0.8, 0.96)])) * W
        v = float(rng.choice([rng.uniform(0.04, 0.2), rng.uniform(0.8, 0.96)])) * H
        tilt, zl, noise = rng.uniform(0.0, 1.0), rng.uniform(2.0, 12.0), rng.uniform(0.0, 0.1)
    else:
        raise ValueError(cls)
    R = _rot([math.pi, 0.0, 0.0]) @ _rot(ax * tilt) @ _rot([0.0, 0.0, spin])
    return R, (u, v), zl, noise


def cases(cls, seed, n):
    """n detectable markers of class ``cls``, drawn from ``seed``."""
    K, D, W, H = CAMERAS[cls]
    rng = np.random.default_rng(seed)
    ids = [0] + sorted(OVERRIDES)
    out = []
    while len(out) < n:
        mid = int(rng.choice(ids))
        L = float(np.float32(OVERRIDES.get(mid, FLEN)))
        R, (u, v), zl, noise = _pose(rng, cls, W, H, L)
        t = zl * L * np.array([(u - K[0, 2]) / K[0, 0], (v - K[1, 2]) / K[1, 1], 1.0])
        c = marker_corners(R, t, K, D, L, rng, noise=noise)
        if detectable(c, W, H):
            out.append(Case(cls, seed, len(out), c, mid, L))
    return out


def oracle(corners, K, D, length, default_len=FLEN):
    """What the reference node publishes for one marker: dict(rvec, tvec, quat xyzw, image_error, object_error, area)."""
    obj = ao.single_marker_object_points(length)
    c = np.asarray(corners, np.float32).reshape(4, 2)
    _, rv, tv = cv2.solvePnP(obj, c, K, D)
    err = ao.reprojection_error(obj, c, K, D, rv, tv)
    f = ao.pose_fields([0], [c], [rv.reshape(3)], [tv.reshape(3)], [err], default_len)[0]
    return dict(rvec=rv.reshape(3), tvec=tv.reshape(3), quat=np.asarray(f["rotation"]), image_error=f["image_error"], object_error=f["object_error"],
                area=f["fiducial_area"])


def reprojection_cost(corners, K, D, length, rvec, tvec) -> float:
    """Sum of squared pixel residuals (float64 projections): what solvePnP minimises."""
    obj = ao.single_marker_object_points(length).astype(np.float64)
    p, _ = cv2.projectPoints(obj, np.asarray(rvec, np.float64), np.asarray(tvec, np.float64), K, D)
    d = p.reshape(4, 2) - np.asarray(corners, np.float64).reshape(4, 2)
    return float(np.sum(d * d))


def gauss_newton(corners, K, D, length, rvec0, tvec0, max_iter=100):
    """Undamped Gauss-Newton on the reprojection error from (rvec0, tvec0), in float64 with cv2.projectPoints' analytic Jacobian,
    run until the step stops shrinking the cost.  Returns (rvec, tvec, cost, iterations)."""
    obj = ao.single_marker_object_points(length).astype(np.float64)
    img = np.asarray(corners, np.float64).reshape(8)
    p = np.concatenate([np.asarray(rvec0, np.float64).reshape(3), np.asarray(tvec0, np.float64).reshape(3)])
    cost = reprojection_cost(corners, K, D, length, p[:3], p[3:])
    it = 0
    for it in range(1, max_iter + 1):
        proj, J = cv2.projectPoints(obj, p[:3].copy(), p[3:].copy(), K, D)
        r = proj.reshape(8) - img
        step, *_ = np.linalg.lstsq(J[:, :6], -r, rcond=None)
        q = p + step
        c = reprojection_cost(corners, K, D, length, q[:3], q[3:])
        if not c < cost:
            break
        p, cost = q, c
        if np.abs(step).max() <= 1e-15 * max(1.0, np.abs(p).max()):
            break
    return p[:3], p[3:], cost, it


def rotation_matrix(rvec):
    return cv2.Rodrigues(np.asarray(rvec, np.float64).reshape(3, 1))[0]


def other_side_of_half_turn(a, b, tol) -> bool:
    """True when rvecs a and b are the same rotation written on the two sides of a half turn: both norms within ``tol`` of pi and
    the rotation matrices within ``tol``.  cv::Rodrigues can return either side there (DESIGN.md, finding 12)."""
    na, nb = np.linalg.norm(a), np.linalg.norm(b)
    return abs(na - math.pi) <= tol and abs(nb - math.pi) <= tol and np.abs(rotation_matrix(a) - rotation_matrix(b)).max() <= tol


TOL = 1e-6


def compare(got, ref, case, K, D, default_len=FLEN):
    """Differences of one published pose against the oracle, as a dict of the quantities the tests bound.  ``half_turn_tie`` marks
    a pose that is the oracle's rotation written on the other side of a half turn (then rvec and quaternion are compared as
    rotations)."""
    tie = bool(np.abs(got["rvec"] - ref["rvec"]).max() > TOL and other_side_of_half_turn(got["rvec"], ref["rvec"], TOL))
    if tie:
        d_rvec = float(np.abs(rotation_matrix(got["rvec"]) - rotation_matrix(ref["rvec"])).max())
        d_quat = float(min(np.abs(got["quat"] - ref["quat"]).max(), np.abs(got["quat"] + ref["quat"]).max()))
    else:
        d_rvec = float(np.abs(got["rvec"] - ref["rvec"]).max())
        d_quat = float(np.abs(got["quat"] - ref["quat"]).max())
    c = np.asarray(case.corners, np.float32).reshape(4, 2)
    de = abs(got["image_error"] - ref["image_error"])
    if de > 1e-6 * ref["image_error"]:
        # getReprojectionError rounds the projections to float32, so a pose 1e-8 away can move one of them by an ulp.  Such a
        # difference is accepted when it is that rounding: the oracle's arithmetic on our own pose gives our value (1e-6), and the
        # difference is within what one ulp per projection can make.
        own = ao.reprojection_error(ao.single_marker_object_points(case.length), c, K, D, np.asarray(got["rvec"], np.float64),
                                    np.asarray(got["tvec"], np.float64))
        ulp = float(np.spacing(np.float32(np.abs(c).max() + 1.0)))
        if abs(got["image_error"] - own) <= 1e-6 * own + 1e-15 and de <= 2.0 * math.sqrt(ref["image_error"]) * ulp + ulp * ulp:
            de = 0.0
    # object_error is image_error scaled by |t| / (diagonal * fiducial_len): that arithmetic on the pose's own image_error
    obj_expect = (got["image_error"] / ao._dist(c[0], c[2])) * (float(np.linalg.norm(got["tvec"])) / default_len)
    return dict(
        half_turn_tie=tie,
        rvec=d_rvec,
        tvec=float(np.abs(got["tvec"] - ref["tvec"]).max()),
        quat=d_quat,
        image_error=de / ref["image_error"] if de > 0.0 else 0.0,
        object_error=abs(got["object_error"] - obj_expect) / max(abs(obj_expect), 1e-300),
        area=abs(got["area"] - ref["area"]) / ref["area"],
    )


def check(diff, what):
    """The tolerances every published pose is held to (image_error 1e-6 relative, object_error and area 1e-9 relative)."""
    assert diff["rvec"] <= TOL and diff["tvec"] <= TOL, (what, diff)
    assert diff["quat"] <= TOL, (what, diff)
    assert diff["image_error"] <= 1e-6, (what, diff)
    assert diff["object_error"] <= 1e-9 and diff["area"] <= 1e-9, (what, diff)
