"""The object-releasing calibration of calib.cuh (host build, tests/hostsim/calib_ro_hostsim.cpp) against
cv2.calibrateCameraROExtended on seeded printed-board problems: boards of 4x3 to 16x12 points, 5 to 60 views, 640x480 to
3840x2160, every distortion preset, the supported flags and a guess, fixed points at 1, n - 2, the top-right corner and the
middle.  Also cv2's behaviour the device call mirrors: what an out-of-range fixed point returns, and the inputs cv2 refuses."""
import cv2
import numpy as np
import pytest

import calib_cases as cc
import calib_ro_cases as rc

G, ZT, PP, K3, AR, FL = (cv2.CALIB_USE_INTRINSIC_GUESS, cv2.CALIB_ZERO_TANGENT_DIST, cv2.CALIB_FIX_PRINCIPAL_POINT, cv2.CALIB_FIX_K3, cv2.CALIB_FIX_ASPECT_RATIO,
                         cv2.CALIB_FIX_FOCAL_LENGTH)


def fixed_of(kind, grid):
    n = grid[0] * grid[1]
    return {"1": 1, "n-2": n - 2, "top-right": grid[0] - 1, "middle": n // 2 + grid[0] // 2}[kind]


# seed, views, grid, size, distortion, flags, fixed point, scale (x, y); five views leave the released problem far from converged
# after cv2's default 30 iterations, where the trajectories of two solvers part at the rounding level: that case runs to convergence
TIGHT = (cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS, 300, 1e-15)
CASES = [
    (1, 5, (8, 6), (640, 480), "zero", 0, "1", (1.004, 1.0)),
    (12, 8, (4, 3), (640, 480), "mild", 0, "top-right", (1.0, 1.004)),
    (2, 10, (6, 4), (1280, 720), "mild", 0, "n-2", (1.0, 1.004)),
    (3, 20, (8, 6), (1920, 1080), "barrel", 0, "top-right", (1.004, 1.004)),
    (4, 60, (5, 4), (3840, 2160), "pincushion", 0, "middle", (1.003, 0.998)),
    (5, 12, (16, 12), (1920, 1080), "mild", 0, "middle", (1.004, 1.0)),
    (6, 15, (7, 5), (1280, 720), "barrel", K3, "top-right", (1.0, 1.004)),
    (7, 15, (7, 5), (1920, 1080), "mild", ZT | PP, "middle", (1.004, 1.0)),
    (8, 15, (7, 5), (1280, 720), "zero", AR | ZT | K3, "1", (1.002, 1.002)),
    (9, 15, (7, 5), (1920, 1080), "pincushion", cv2.CALIB_FIX_K1 | cv2.CALIB_FIX_K2, "n-2", (1.004, 1.0)),
    (10, 15, (7, 5), (1920, 1080), "barrel", G, "top-right", (1.004, 1.0)),
    (11, 15, (7, 5), (1920, 1080), "mild", G | FL | K3, "middle", (1.0, 1.004)),
]


def _guess(flags, K, D):
    if flags & G:
        return K * np.array([[1.01, 1, 1.003], [1, 0.99, 0.997], [1, 1, 1]]), D * 0.9
    return (K, None) if flags & AR else (None, None)


@pytest.mark.parametrize("case", CASES, ids=[str(c[0]) for c in CASES])
def test_host_matches_cv2(case):
    seed, nv, grid, size, dist, flags, kind, scale = case
    O, I, K, D, true = rc.make_printed_problem(seed, nv, grid, size, dist, 0.2, scale)
    fixed = fixed_of(kind, grid)
    Kg, Dg = _guess(flags, K, D)
    crit = TIGHT if nv < 6 else None
    hs = rc.hs_calibrate_ro(O, I, size, fixed, Kg, Dg, flags, crit)
    assert hs["status"] == 0
    ref = rc.cv2_calibrate_ro(O, I, size, fixed, Kg, Dg, flags, crit)
    rc.assert_matches_cv2_ro(hs, ref, O, fixed, "case %d" % seed)
    assert hs["iterations"] >= 1 and len(hs["steps"]) >= hs["iterations"]


def test_release_lowers_rms_and_recovers_the_print_scale():
    """The point of the method: on a board printed 0.4 % too tall, the released fit has a lower rms than the standard one and its
    new points carry the scale (relative to the fixed points 0 and the top-right corner, which pin the x extent)."""
    grid = (9, 6)
    O, I, K, D, true = rc.make_printed_problem(21, 25, grid, (1920, 1080), "mild", 0.2, (1.0, 1.004), bow=0.0, jitter=0.0)
    fixed = grid[0] - 1
    hs = rc.hs_calibrate_ro(O, I, (1920, 1080), fixed)
    std = cc.hs_calibrate(O, I, (1920, 1080))
    assert hs["rms"] < 0.9 * std["rms"]  # 0.2 px of image noise is the floor of both
    new = hs["new_obj"].astype(np.float64)
    ext_y = new[:, 1].max() - new[:, 1].min()
    ext_x = new[:, 0].max() - new[:, 0].min()
    nominal = O[0]
    aspect = (ext_y / ext_x) / ((np.ptp(nominal[:, 1])) / (np.ptp(nominal[:, 0])))
    assert abs(aspect - 1.004) < 5e-4, aspect


def test_out_of_range_fixed_point_is_the_standard_calibration():
    """cv2 releases nothing for fixed points 0, n - 1 and -1: the standard calibration's result and no new points; the host build
    of the standard calibration (calib_hostsim.cpp) matches it as it matches calibrateCameraExtended."""
    O, I, K, D, true = rc.make_printed_problem(31, 8, (5, 4), (1280, 720), "mild", 0.2)
    n = len(O[0])
    std = cc.cv2_calibrate(O, I, (1280, 720))
    hs = cc.hs_calibrate(O, I, (1280, 720))
    for fixed in (0, n - 1, -1, n, 10 * n):
        ref = rc.cv2_calibrate_ro(O, I, (1280, 720), fixed)
        assert ref["new_obj"] is None and ref["std_obj"] is None
        assert ref["rms"] == std["rms"] and np.array_equal(ref["K"], std["K"]) and np.array_equal(ref["std_ext"], std["std_ext"])
        cc.assert_matches_cv2(hs, ref, "fixed %d" % fixed)


def test_cv2_refusals():
    """The inputs fid_calibrate_camera_ro refuses (FID_CALIB_E_RO_VIEWS, FID_CALIB_E_NONPLANAR) are the ones cv2 raises on."""
    O, I, K, D, true = rc.make_printed_problem(41, 6, (5, 4), (1280, 720), "mild", 0.2)
    fixed = 4
    unequal_O, unequal_I = [O[0][:-1]] + O[1:], [I[0][:-1]] + I[1:]
    with pytest.raises(cv2.error, match="should be equal"):
        rc.cv2_calibrate_ro(unequal_O, unequal_I, (1280, 720), fixed)
    moved = [o.copy() for o in O]
    moved[3][7, 0] += np.float32(1e-3)
    with pytest.raises(cv2.error, match="should be identical"):
        rc.cv2_calibrate_ro(moved, I, (1280, 720), fixed)
    bowed = [true.astype(np.float32) for _ in O]
    with pytest.raises(cv2.error, match="non-planar"):
        rc.cv2_calibrate_ro(bowed, I, (1280, 720), fixed)
    # the same board with a guess runs, and the host build follows it
    hs = rc.hs_calibrate_ro(bowed, I, (1280, 720), fixed, K, D, G)
    ref = rc.cv2_calibrate_ro(bowed, I, (1280, 720), fixed, K, D, G)
    rc.assert_matches_cv2_ro(hs, ref, bowed, fixed, "bowed with a guess")


def test_host_matches_the_stored_cv2_result_of_a_large_board():
    """384 points x 30 views (m = 1 161), too slow for cv2 on every run: cv2's stored result (tests/golden/calib_ro_384x30.npz)."""
    O, I, size, fixed, ref = rc.golden()
    hs = rc.hs_calibrate_ro(O, I, size, fixed)
    assert hs["status"] == 0
    rc.assert_matches_cv2_ro(hs, ref, O, fixed, "384 x 30")


def test_degenerate_inputs():
    """What cv2 does where the released problem is degenerate.  With as many free parameters as residuals cv2 raises ("There
    should be less vars to optimize ..."); fid_calibrate_camera_ro refuses with FID_CALIB_E_RO_RESIDUALS.  With every view the
    same image (no baseline: the depth of every point along its ray is free) cv2 fits the points exactly (rms ~ 0) and inverts
    the singular J^T J by SVD; the Cholesky of the reduced system meets a non-positive pivot and the library returns
    FID_CALIB_E_RO_SINGULAR (8) instead of a result."""
    O, I, K, D, true = rc.make_printed_problem(51, 1, (5, 4), (1280, 720), "mild", 0.2)
    with pytest.raises(cv2.error, match="less vars to optimize"):
        rc.cv2_calibrate_ro(O, I, (1280, 720), 4)
    O, I, K, D, true = rc.make_printed_problem(52, 4, (5, 4), (1280, 720), "mild", 0.2)
    same = [I[0]] * 4
    ref = rc.cv2_calibrate_ro(O, same, (1280, 720), 4)
    assert ref["rms"] < 1e-9 and np.all(np.isfinite(ref["std_obj"]))
    assert rc.hs_calibrate_ro(O, same, (1280, 720), 4)["status"] == 8
