"""Seeded printed-board problems for the object-releasing calibration (cv2.calibrateCameraROExtended), the cv2 oracle, and the host
build of calib.cuh's release path (tests/hostsim/calib_ro_hostsim.cpp, compiled with g++ into a temporary directory once per
session, as calib_cases.py compiles calib_hostsim.cpp).

A printed board differs from its nominal geometry: the printer scales it (anisotropically, by a few tenths of a percent), the sheet
bows out of its plane, and every printed point sits a little off.  The views see the true board; the calibration is given the
nominal one."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import cv2
import numpy as np

import calib_cases as cc

_HERE = os.path.dirname(os.path.abspath(__file__))
_harness = None
_vp = C.c_void_p


def _p(a):
    return a.ctypes.data_as(_vp)


def harness():
    global _harness
    if _harness is None:
        tmp = tempfile.mkdtemp(prefix="fid_calib_ro_hostsim_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "libfid_calib_ro_hostsim.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, os.path.join(_HERE, "hostsim", "calib_ro_hostsim.cpp")])
        _harness = C.CDLL(so)
        _harness.hs_calibrate_ro.argtypes = [C.c_int, C.c_int, _vp, _vp, C.c_int, C.c_int, _vp, _vp, C.c_int, C.c_int, C.c_int, C.c_double] + [_vp] * 8
    return _harness


def hs_calibrate_ro(O, I, size, fixed, K=None, D=None, flags=0, criteria=None):
    """The release path of calib.cuh on the host (a released input only): hs_calibrate's dict plus new_obj [n][3] (float32) and
    std_obj [n][3]."""
    nv, n = len(O), len(O[0])
    obj = np.ascontiguousarray(O[0], np.float32).reshape(-1, 3)
    img = np.ascontiguousarray(np.concatenate(I), np.float32).reshape(-1, 2)
    out = np.zeros(23)
    rv, tv, se, pve = np.zeros((nv, 3)), np.zeros((nv, 3)), np.zeros((nv, 6)), np.zeros(nv)
    steps = np.zeros(2048, np.uint8)
    new_obj, std_obj = np.zeros((n, 3), np.float32), np.zeros((n, 3))
    Ka = None if K is None else np.ascontiguousarray(K, np.float64).reshape(9)
    Da = None if (K is None and D is None) else np.ascontiguousarray(np.r_[np.zeros(0) if D is None else np.ravel(D), np.zeros(5)][:5], np.float64)
    max_iter, eps = cc.criteria_of(criteria)
    st = harness().hs_calibrate_ro(nv, n, _p(obj), _p(img), int(size[0]), int(size[1]), None if Ka is None else _p(Ka), None if Da is None else _p(Da), int(flags),
                                   int(fixed), max_iter, eps, _p(out), _p(rv), _p(tv), _p(se), _p(pve), _p(steps), _p(new_obj), _p(std_obj))
    Kout = np.array([[out[1], 0, out[3]], [0, out[2], out[4]], [0, 0, 1]])
    return dict(status=st, rms=out[0], K=Kout, D=out[5:10].copy(), rvecs=rv, tvecs=tv, std_int=out[10:19].copy(), std_ext=se, pve=pve, iterations=int(out[19]),
                steps=steps[: int(out[20])].copy(), new_obj=new_obj, std_obj=std_obj)


def cv2_calibrate_ro(O, I, size, fixed, K=None, D=None, flags=0, criteria=None):
    """cv2.calibrateCameraROExtended in the same dict form (raises cv2.error where cv2 does); new_obj / std_obj are None when
    cv2 releases nothing."""
    kw = {} if criteria is None else {"criteria": criteria}
    r = cv2.calibrateCameraROExtended([np.asarray(o, np.float32).reshape(-1, 3) for o in O], [np.asarray(i, np.float32).reshape(-1, 2) for i in I], tuple(size),
                                      int(fixed), None if K is None else np.array(K, np.float64), None if D is None else np.array(D, np.float64).reshape(1, -1),
                                      flags=flags, **kw)
    rms, Ko, Do, rv, tv, newobj, sdi, sde, sdo, pv = r
    return dict(rms=rms, K=Ko, D=Do.ravel()[:5], rvecs=np.array(rv).reshape(-1, 3), tvecs=np.array(tv).reshape(-1, 3), std_int=sdi.ravel()[:9], std_ext=sde.reshape(-1, 6),
                pve=pv.ravel(), new_obj=None if newobj is None else newobj.reshape(-1, 3), std_obj=None if sdo is None else sdo.reshape(-1, 3), raw=r)


def assert_matches_cv2_ro(got, ref, O, fixed, what="", std_tol=1e-4, rms_tol=1e-9):
    """calib_cases.assert_matches_cv2's bounds, and every new board coordinate within 1e-4 of cv2's standard deviation for it,
    the standard deviations of the coordinates within std_tol relative, and the seven fixed coordinates equal to the input with a
    standard deviation of exactly 0."""
    cc.assert_matches_cv2(got, ref, what, std_tol, rms_tol)
    n = len(O[0])
    free = np.ones((n, 3), bool)
    free[0] = free[fixed] = False
    free[n - 1, 2] = False
    so = ref["std_obj"]
    assert np.all((so > 0) == free), (what, np.argwhere((so > 0) != free))
    d = np.abs(got["new_obj"].astype(np.float64) - ref["new_obj"].astype(np.float64))
    # float32 outputs: one unit in the last place of the coordinate is allowed on top of the bound
    ulp = np.spacing(np.abs(ref["new_obj"])).astype(np.float64)
    assert np.all(d[free] <= 1e-4 * so[free] + ulp[free]), (what, (d / np.where(free, so, 1)).max())
    board = np.asarray(O[0], np.float32).reshape(-1, 3)
    assert np.array_equal(got["new_obj"][~free], board[~free]) and np.all(got["std_obj"][~free] == 0), what
    assert np.all(np.abs(got["std_obj"][free] / so[free] - 1) <= std_tol), (what, np.abs(got["std_obj"][free] / so[free] - 1).max())


def make_printed_problem(seed, n_views, grid=(6, 4), size=(1920, 1080), dist="mild", noise=0.1, scale=(1.004, 1.0), bow=1e-3, jitter=2e-4, square=0.04):
    """calib_cases.make_problem's views of a printed grid: the true board is the nominal one scaled by `scale` in x and y, bowed
    out of its plane (z up to `bow` metres at the centre) and jittered per point (`jitter` metres, every axis).  Every view
    holds every point.  Returns (nominal object points per view, image points, K, D, true board)."""
    rng = np.random.default_rng(seed)
    gx, gy = grid
    nominal = np.array([[(x + 1) * square, (y + 1) * square, 0] for y in range(gy) for x in range(gx)], np.float32)
    ctr = nominal.mean(0)
    half = np.maximum(np.abs(nominal - ctr).max(0), 1e-9)
    u = (nominal[:, :2] - ctr[:2]) / half[:2]
    true = nominal.astype(np.float64).copy()
    true[:, 0] = ctr[0] + (true[:, 0] - ctr[0]) * scale[0]
    true[:, 1] = ctr[1] + (true[:, 1] - ctr[1]) * scale[1]
    true[:, 2] = bow * (1 - 0.5 * (u ** 2).sum(1))
    true += rng.normal(0, jitter, true.shape)
    O, I, K, D = cc.make_problem(seed, n_views, grid, size, dist, 0.0, 0.0, square)
    # the same seeded poses, re-projected through the true board with fresh noise
    I2 = []
    for o, m in zip(O, I):
        ok, rv, tv = cv2.solvePnP(o.astype(np.float64), m.astype(np.float64), K, D, flags=cv2.SOLVEPNP_ITERATIVE)
        p, _ = cv2.projectPoints(true, rv, tv, K, D)
        I2.append((p.reshape(-1, 2) + rng.normal(0, noise, (len(o), 2))).astype(np.float32))
    return [nominal.copy() for _ in O], I2, K, D, true


def golden(name="calib_ro_384x30.npz"):
    """A stored cv2.calibrateCameraROExtended result (tests/golden/make_calib_ro_golden.py): (object points per view, image points,
    image size, fixed point, cv2's result in cv2_calibrate_ro's dict form)."""
    z = np.load(os.path.join(_HERE, "golden", name))
    O = [z["board"].copy() for _ in range(len(z["img"]))]
    I = [m.copy() for m in z["img"]]
    ref = {k: z[k] for k in ("K", "D", "rvecs", "tvecs", "std_int", "std_ext", "pve", "new_obj", "std_obj")}
    ref["rms"] = float(z["rms"])
    return O, I, tuple(int(v) for v in z["size"]), int(z["fixed"]), ref
