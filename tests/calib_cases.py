"""Seeded calibration problems, the cv2.calibrateCameraExtended oracle, and the host build of fiducials_b200/csrc/calib.cuh
(tests/hostsim/calib_hostsim.cpp, compiled with g++ into a temporary directory once per session)."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import cv2
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_harness = None
_vp = C.c_void_p


def _p(a):
    return a.ctypes.data_as(_vp)


def harness():
    global _harness
    if _harness is None:
        tmp = tempfile.mkdtemp(prefix="fid_calib_hostsim_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "libfid_calib_hostsim.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, os.path.join(_HERE, "hostsim", "calib_hostsim.cpp")])
        _harness = C.CDLL(so)
        _harness.hs_calibrate.argtypes = [C.c_int, _vp, _vp, _vp, C.c_int, C.c_int, _vp, _vp, C.c_int, C.c_int, C.c_double, _vp, _vp, _vp, _vp, _vp, _vp]
    return _harness


def criteria_of(criteria):
    """CvLevMarq's max_iter and epsilon of a cv2 criteria tuple (None = cv2's default)."""
    if criteria is None:
        return 30, np.finfo(np.float64).eps
    t, it, eps = criteria
    return (min(max(int(it), 1), 1000) if t & 1 else 30), (max(float(eps), 0.0) if t & 2 else np.finfo(np.float64).eps)


def hs_calibrate(O, I, size, K=None, D=None, flags=0, criteria=None):
    """calib.cuh on the host: a dict of status, rms, K, D, rvecs, tvecs, std_int (9), std_ext [n][6], pve [n], iterations, steps."""
    nv = len(O)
    off = np.zeros(nv + 1, np.int32)
    off[1:] = np.cumsum([len(o) for o in O])
    obj = np.ascontiguousarray(np.concatenate(O), np.float32).reshape(-1, 3)
    img = np.ascontiguousarray(np.concatenate(I), np.float32).reshape(-1, 2)
    out = np.zeros(23)
    rv, tv, se, pve = np.zeros((nv, 3)), np.zeros((nv, 3)), np.zeros((nv, 6)), np.zeros(nv)
    steps = np.zeros(2048, np.uint8)
    Ka = None if K is None else np.ascontiguousarray(K, np.float64).reshape(9)
    Da = None if (K is None and D is None) else np.ascontiguousarray(np.r_[np.zeros(0) if D is None else np.ravel(D), np.zeros(5)][:5], np.float64)
    max_iter, eps = criteria_of(criteria)
    st = harness().hs_calibrate(nv, _p(off), _p(obj), _p(img), int(size[0]), int(size[1]), None if Ka is None else _p(Ka), None if Da is None else _p(Da), int(flags),
                                max_iter, eps, _p(out), _p(rv), _p(tv), _p(se), _p(pve), _p(steps))
    Kout = np.array([[out[1], 0, out[3]], [0, out[2], out[4]], [0, 0, 1]])
    return dict(status=st, rms=out[0], K=Kout, D=out[5:10].copy(), rvecs=rv, tvecs=tv, std_int=out[10:19].copy(), std_ext=se, pve=pve, iterations=int(out[19]),
                steps=steps[: int(out[20])].copy())


def cv2_calibrate(O, I, size, K=None, D=None, flags=0, criteria=None):
    """cv2.calibrateCameraExtended in the same dict form (raises cv2.error where cv2 does)."""
    kw = {} if criteria is None else {"criteria": criteria}
    r = cv2.calibrateCameraExtended([np.asarray(o, np.float32).reshape(-1, 3) for o in O], [np.asarray(i, np.float32).reshape(-1, 2) for i in I], tuple(size),
                                    None if K is None else np.array(K, np.float64), None if D is None else np.array(D, np.float64).reshape(1, -1), flags=flags, **kw)
    rms, Ko, Do, rv, tv, sdi, sde, pv = r
    return dict(rms=rms, K=Ko, D=Do.ravel()[:5], rvecs=np.array(rv).reshape(-1, 3), tvecs=np.array(tv).reshape(-1, 3), std_int=sdi.ravel()[:9],
                std_int18=sdi.ravel(), std_ext=sde.reshape(-1, 6), pve=pv.ravel())


def intrinsics(d):
    K = d["K"]
    return np.r_[K[0, 0], K[1, 1], K[0, 2], K[1, 2], np.ravel(d["D"])[:5]]


def assert_matches_cv2(got, ref, what="", std_tol=1e-4, rms_tol=1e-9):
    """rms within rms_tol relative, every parameter within 1e-4 of cv2's standard deviation for it (fixed parameters equal to 1e-9
    relative), standard deviations within std_tol relative and per-view errors within 1e-6 relative."""
    assert abs(got["rms"] / ref["rms"] - 1) <= rms_tol, (what, got["rms"], ref["rms"])
    si = ref["std_int"]
    free = si > 0
    gi, ri = intrinsics(got), intrinsics(ref)
    assert np.all(np.abs(gi - ri)[free] <= 1e-4 * si[free]), (what, (gi - ri) / np.where(free, si, 1))
    assert np.all(np.abs(gi - ri)[~free] <= 1e-9 * np.maximum(np.abs(ri[~free]), 1)), (what, gi, ri)
    se = ref["std_ext"]
    assert np.all(np.abs(got["rvecs"] - ref["rvecs"]) <= 1e-4 * se[:, :3]), (what, np.abs(got["rvecs"] - ref["rvecs"]) / se[:, :3])
    assert np.all(np.abs(got["tvecs"] - ref["tvecs"]) <= 1e-4 * se[:, 3:]), (what, np.abs(got["tvecs"] - ref["tvecs"]) / se[:, 3:])
    assert np.all(got["std_int"][~free] == 0)
    assert np.all(np.abs(got["std_int"][free] / si[free] - 1) <= std_tol), (what, got["std_int"] / np.where(free, si, 1) - 1)
    assert np.all(np.abs(got["std_ext"] / se - 1) <= std_tol), (what, np.abs(got["std_ext"] / se - 1).max())
    assert np.all(np.abs(got["pve"] / ref["pve"] - 1) <= 1e-6), (what, np.abs(got["pve"] / ref["pve"] - 1).max())
    return (np.abs(gi - ri)[free] / si[free]).max(), np.abs(got["std_ext"] / se - 1).max()


def cv2_converged(O, I, size, K=None, D=None, flags=0, criteria=None):
    """cv2's result, and whether it equals its (COUNT + EPS, 300, 1e-16) result (converged to the least-squares minimum)."""
    ref = cv2_calibrate(O, I, size, K, D, flags, criteria)
    tight = cv2_calibrate(O, I, size, K, D, flags, (cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS, 300, 1e-16))
    same = abs(ref["rms"] / tight["rms"] - 1) < 1e-12 and np.allclose(intrinsics(ref), intrinsics(tight), rtol=1e-10, atol=0)
    return ref, same


# ---- the seeded problems ------------------------------------------------------------------------------------------------------
SIZES = [(640, 480), (1280, 720), (1920, 1080), (3840, 2160)]
DISTORTIONS = {"zero": np.zeros(5), "barrel": np.array([-0.28, 0.09, 0.0008, -0.0006, -0.01]), "mild": np.array([-0.12, 0.05, 0.001, -0.0008, 0.0]),
               "pincushion": np.array([0.18, -0.05, -0.0005, 0.0007, 0.01])}


def _rot(r):
    return cv2.Rodrigues(np.asarray(r, np.float64))[0]


def make_problem(seed, n_views, grid=(6, 4), size=(1920, 1080), dist="mild", noise=0.1, partial=0.0, square=0.04):
    """n_views views of a planar grid of (gx x gy) points (ChArUco corners of a (gx+1) x (gy+1) board) seen from seeded poses that
    keep every point inside the image; with `partial` > 0 a random share of the views keeps only a random subset of its points
    (at least 4, never collinear), as occlusion leaves them.  Returns (object points, image points, K, D)."""
    rng = np.random.default_rng(seed)
    W, H = size
    f = W * rng.uniform(0.65, 0.95)
    K = np.array([[f, 0, W / 2 + rng.uniform(-0.03, 0.03) * W], [0, f * rng.uniform(0.98, 1.02), H / 2 + rng.uniform(-0.03, 0.03) * H], [0, 0, 1]])
    D = DISTORTIONS[dist] if isinstance(dist, str) else np.asarray(dist, np.float64)
    gx, gy = grid
    obj = np.array([[(x + 1) * square, (y + 1) * square, 0] for y in range(gy) for x in range(gx)], np.float32)
    ctr = np.array([(gx + 1) * square / 2, (gy + 1) * square / 2, 0])
    ext = max(gx + 1, gy + 1) * square
    O, I = [], []
    tries = 0
    while len(O) < n_views:
        tries += 1
        assert tries < 200 * n_views + 1000
        r = rng.normal(0, 0.35, 3)
        R = _rot(r)
        z = ext * f / (W * rng.uniform(0.35, 0.9))
        t = np.array([rng.uniform(-0.25, 0.25) * z * W / f, rng.uniform(-0.25, 0.25) * z * H / f, z]) - R @ ctr
        rv = cv2.Rodrigues(R)[0]
        p, _ = cv2.projectPoints(obj.astype(np.float64), rv, t, K, D)
        p = p.reshape(-1, 2)
        cam = (obj.astype(np.float64) @ R.T) + t
        if (cam[:, 2] <= 0).any() or (p[:, 0] < 0).any() or (p[:, 0] > W - 1).any() or (p[:, 1] < 0).any() or (p[:, 1] > H - 1).any():
            continue
        p = p + rng.normal(0, noise, p.shape)
        keep = np.arange(len(obj))
        if partial and rng.uniform() < partial:
            while True:
                keep = np.sort(rng.choice(len(obj), int(rng.integers(4, len(obj) + 1)), replace=False))
                g = np.stack([keep % gx, keep // gx], 1)
                d = g[1:] - g[0]
                if np.any(d[:, 0, None] * d[None, :, 1] - d[:, 1, None] * d[None, :, 0]):
                    break
        O.append(obj[keep].copy())
        I.append(p[keep].astype(np.float32))
    return O, I, K, D
