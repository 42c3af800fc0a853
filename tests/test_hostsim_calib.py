"""Camera calibration (fiducials_b200/csrc/calib.cuh, compiled for the host from tests/hostsim/calib_hostsim.cpp) against
cv2.calibrateCameraExtended over a seeded sweep, and the input checks of fid_calibrate_camera, which run before it looks for a
device.  CPU only."""
import ctypes as C

import cv2
import numpy as np
import pytest

import calib_cases as cc
from fiducials_b200 import calib

G = cv2.CALIB_USE_INTRINSIC_GUESS
_worst = {"param/sigma": 0.0, "std": 0.0}

# (seed, views, grid, size, distortion, noise px, partial share, flags, guess, criteria)
SWEEP = [
    (1, 3, (6, 4), (640, 480), "zero", 0.0, 0.0, 0, False, None),
    (2, 5, (6, 4), (1280, 720), "mild", 0.1, 0.5, 0, False, None),
    (3, 12, (6, 4), (1920, 1080), "barrel", 0.3, 0.3, 0, False, None),
    (4, 20, (11, 8), (3840, 2160), "pincushion", 0.5, 0.5, 0, False, None),
    (5, 40, (6, 4), (1920, 1080), "mild", 0.2, 0.6, 0, False, None),
    (6, 100, (6, 4), (1280, 720), "barrel", 0.1, 0.4, 0, False, None),
    (7, 6, (32, 32), (3840, 2160), "mild", 0.2, 0.0, 0, False, None),
    (8, 8, (2, 2), (640, 480), "zero", 0.05, 0.0, 0, False, None),  # 4 points per view
    (9, 10, (6, 4), (1920, 1080), "mild", 0.1, 0.3, cv2.CALIB_FIX_ASPECT_RATIO, False, None),
    (10, 10, (6, 4), (1920, 1080), "barrel", 0.1, 0.3, cv2.CALIB_FIX_PRINCIPAL_POINT, False, None),
    (11, 10, (6, 4), (1280, 720), "mild", 0.1, 0.3, cv2.CALIB_ZERO_TANGENT_DIST, False, None),
    (12, 10, (6, 4), (1920, 1080), "mild", 0.1, 0.3, cv2.CALIB_FIX_FOCAL_LENGTH, False, None),
    (13, 10, (6, 4), (1920, 1080), "barrel", 0.2, 0.3, cv2.CALIB_FIX_K1, False, None),
    (14, 10, (6, 4), (1920, 1080), "barrel", 0.2, 0.3, cv2.CALIB_FIX_K2, False, None),
    (15, 10, (6, 4), (1920, 1080), "mild", 0.2, 0.3, cv2.CALIB_FIX_K3, False, None),
    (16, 15, (9, 6), (1920, 1080), "zero", 0.1, 0.3, cv2.CALIB_FIX_K3 | cv2.CALIB_ZERO_TANGENT_DIST, False, None),
    (17, 15, (9, 6), (1280, 720), "mild", 0.1, 0.3, cv2.CALIB_FIX_ASPECT_RATIO | cv2.CALIB_FIX_PRINCIPAL_POINT | cv2.CALIB_FIX_K3, False, None),
    (18, 12, (6, 4), (1920, 1080), "barrel", 0.2, 0.3, G, True, None),
    (19, 12, (6, 4), (1920, 1080), "pincushion", 0.2, 0.3, G | cv2.CALIB_FIX_FOCAL_LENGTH | cv2.CALIB_FIX_PRINCIPAL_POINT, True, None),
    (20, 12, (6, 4), (1920, 1080), "mild", 0.2, 0.3, G | cv2.CALIB_FIX_ASPECT_RATIO | cv2.CALIB_FIX_K1 | cv2.CALIB_FIX_K2, True, None),
    (21, 12, (6, 4), (1920, 1080), "mild", 0.2, 0.3, 0, False, (cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS, 100, 1e-12)),
    (22, 12, (6, 4), (1920, 1080), "mild", 0.2, 0.3, 0, False, (cv2.TERM_CRITERIA_COUNT, 40, 0)),
    (23, 25, (11, 8), (1920, 1080), "barrel", 0.4, 0.7, 0, False, None),
]


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\ncalibration vs cv2: max |d param| / cv2 sigma = %.3g, max relative d std = %.3g" % (_worst["param/sigma"], _worst["std"]))


def _guess(K, D, rng):
    Kg = K.copy()
    Kg[0, 0] *= rng.uniform(0.97, 1.03)
    Kg[1, 1] = Kg[0, 0] * K[1, 1] / K[0, 0]
    Kg[0, 2] += rng.uniform(-10, 10)
    Kg[1, 2] += rng.uniform(-10, 10)
    return Kg, np.asarray(D) * rng.uniform(0.8, 1.2)


@pytest.mark.parametrize("case", SWEEP, ids=[str(c[0]) for c in SWEEP])
def test_calibration_matches_cv2(case):
    seed, nv, grid, size, dist, noise, partial, flags, guess, crit = case
    O, I, K, D = cc.make_problem(seed, nv, grid, size, dist, noise, partial)
    rng = np.random.default_rng(seed + 1000)
    Kg, Dg = _guess(K, D, rng) if guess else (K if flags & cv2.CALIB_FIX_ASPECT_RATIO else None, None)
    ref, converged = cc.cv2_converged(O, I, size, Kg, Dg, flags, crit)
    got = cc.hs_calibrate(O, I, size, Kg, Dg, flags, crit)
    assert got["status"] == 0
    assert converged, "cv2 did not converge: the case checks nothing"
    # a focal length fixed at the initial estimate: the two initial estimates differ in the last digits (findHomography's LM stops
    # after 10 iterations, before the rounding of its solve settles), and the minimum given that focal length moves with it
    fixed_init = flags & cv2.CALIB_FIX_FOCAL_LENGTH and not guess
    dp, ds = cc.assert_matches_cv2(got, ref, "case %d" % seed, rms_tol=1e-7 if fixed_init else 1e-9)
    _worst["param/sigma"] = max(_worst["param/sigma"], dp)
    _worst["std"] = max(_worst["std"], ds)
    assert 1 <= got["iterations"] <= cc.criteria_of(crit)[0] and got["steps"].sum() == got["iterations"]


@pytest.mark.parametrize("k", [1, 2, 3, 4, 5])
def test_first_iterations_follow_cv2(k):
    """With (COUNT, k) both stop after k iterations: the initial estimate and the first steps agree with cv2's, to the rounding of
    their different linear solves (cv2 solves the dense system by SVD)."""
    O, I, K, D = cc.make_problem(31, 12, (6, 4), (1920, 1080), "mild", 0.1, 0.3)
    got = cc.hs_calibrate(O, I, (1920, 1080), criteria=(cv2.TERM_CRITERIA_COUNT, k, 0))
    ref = cc.cv2_calibrate(O, I, (1920, 1080), criteria=(cv2.TERM_CRITERIA_COUNT, k, 0))
    assert got["iterations"] == k
    assert abs(got["rms"] / ref["rms"] - 1) <= 1e-5
    assert np.abs(cc.intrinsics(got) - cc.intrinsics(ref)).max() <= 1e-3 * np.abs(cc.intrinsics(ref)).max()


def test_one_view_is_accepted():
    """cv2 accepts a single view (and returns a poorly determined camera); so does the library, from the same start."""
    O, I, K, D = cc.make_problem(41, 1, (6, 4), (1920, 1080), "mild", 0.1)
    got = cc.hs_calibrate(O, I, (1920, 1080))
    ref = cc.cv2_calibrate(O, I, (1920, 1080))
    assert got["status"] == 0 and np.isfinite(got["rms"])
    assert abs(got["rms"] - ref["rms"]) <= 1e-3 * max(ref["rms"], 1e-3)


def test_collinear_view_raises_like_cv2():
    O, I, K, D = cc.make_problem(42, 5, (6, 4), (1920, 1080), "mild", 0.1)
    O[2], I[2] = O[2][:6], I[2][:6]  # one row of the grid: collinear
    with pytest.raises(cv2.error):
        cc.cv2_calibrate(O, I, (1920, 1080))
    assert cc.hs_calibrate(O, I, (1920, 1080))["status"] == 3  # FID_CALIB_E_HOMOGRAPHY


def _api(O, I, size=(1920, 1080), K=None, D=None, flags=0):
    """fid_calibrate_camera's status and result status (the input is checked before any device is looked for)."""
    from fiducials_b200 import _lib

    lib = _lib.load()
    off, obj, img = calib._views(O, I)
    res = _lib.fid_calib_result()
    guess = None
    if K is not None:
        guess = _lib.fid_camera()
        for i in range(9):
            guess.K[i] = float(np.ravel(K)[i])
        for i in range(5):
            guess.D[i] = float(np.ravel(D)[i]) if D is not None else 0.0
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    st = lib.fid_calibrate_camera(0, len(O), vp(off), vp(obj), vp(img), size[0], size[1], None if guess is None else C.byref(guess), flags, None, C.byref(res), None,
                                  None, None, None, None)
    return st, res.status


def test_input_checks_mirror_cv2():
    import torch

    O, I, K, D = cc.make_problem(43, 5, (6, 4), (1920, 1080), "mild", 0.1)
    ok = -2 if not torch.cuda.is_available() else 0  # FID_ERR_NO_DEVICE past the checks on a machine without a GPU
    assert _api(O, I)[0] == ok
    # fewer than 4 points in a view
    O3, I3 = list(O), list(I)
    O3[1], I3[1] = O[1][:3], I[1][:3]
    with pytest.raises(cv2.error):
        cc.cv2_calibrate(O3, I3, (1920, 1080))
    assert _api(O3, I3) == (-1, 1)
    # an object plane at z = 0.01 is not planar without a guess
    Oz = [o.copy() for o in O]
    for o in Oz:
        o[:, 2] = 0.01
    with pytest.raises(cv2.error):
        cc.cv2_calibrate(Oz, I, (1920, 1080))
    assert _api(Oz, I) == (-1, 2)
    # the guess: principal point outside the image, non-positive focal length
    for bad in ([[1400, 0, 2000], [0, 1400, 540], [0, 0, 1]], [[-5, 0, 960], [0, 1400, 540], [0, 0, 1]]):
        with pytest.raises(cv2.error):
            cc.cv2_calibrate(O, I, (1920, 1080), np.array(bad, float), np.zeros(5), G)
        assert _api(O, I, K=np.array(bad, float), flags=G) == (-1, 4)
    # non-finite points
    In = [i.copy() for i in I]
    In[0][0, 0] = np.nan
    assert _api(O, In) == (-1, 6)
    # other camera models are not fid_camera's
    for fl in (cv2.CALIB_RATIONAL_MODEL, cv2.CALIB_THIN_PRISM_MODEL, cv2.CALIB_TILTED_MODEL, cv2.CALIB_FIX_K4, cv2.CALIB_USE_LU):
        assert _api(O, I, flags=fl)[0] == -4


def test_charuco_views():
    from fiducials_b200.board import charuco_board

    b = charuco_board((7, 5), 0.04, 0.03)
    ids = [np.array([0, 1, 2, 3, 7, 8]), np.array([0, 1, 2, 3, 4, 5]), np.array([5, 11, 17]), np.array([23, 12, 4, 19])]
    xy = [np.random.default_rng(i).uniform(0, 500, (len(c), 2)) for i, c in enumerate(ids)]
    O, I, kept = calib.charuco_views(b, ids, xy)
    assert kept == [0, 3]  # frame 1: one row (collinear), frame 2: 3 corners
    ref = cv2.aruco.CharucoBoard((7, 5), 0.04, 0.03, cv2.aruco.getPredefinedDictionary(cv2.aruco.DICT_6X6_250))
    for k, f in enumerate(kept):
        ro, ri = ref.matchImagePoints(np.asarray(xy[f], np.float32).reshape(-1, 1, 2), ids[f].reshape(-1, 1).astype(np.int32))
        assert np.array_equal(O[k], ro.reshape(-1, 3)) and np.array_equal(I[k], ri.reshape(-1, 2))
