"""fid_calibrate_camera_ro on the device against the host build of calib.cuh's release path (the same numbers to the rounding of
the reduced system's tensor-core sums) and against cv2.calibrateCameraROExtended; runs over several chunks of views (600 views)
and at the caps' scale (1 024 points x 1 000 views); cv2's stored result for 384 points x 30 views; the standard path for
out-of-range fixed points; the refusals; and end to end from rendered ChArUco frames of a board printed 0.4 % taller than wide."""
import cv2
import numpy as np
import pytest

import calib_cases as cc
import calib_ro_cases as rc
from fiducials_b200 import _lib, calib

pytestmark = pytest.mark.gpu

# device against host: the reduced system is summed in another order on the tensor cores (and factored blockwise), so values
# agree to rounding amplified by its condition, not bit for bit; measured on an H100: 3.5e-7 relative at most over
# the cases below (small rvec components), 4e-11 on most
HOST_TOL = 1e-6


def _device(O, I, size, fixed, K=None, D=None, flags=0, criteria=None):
    st = _lib.fid_calib_stats()
    r = calib.calibrate_camera_ro(O, I, size, fixed, K, D, flags, criteria, stats=st)
    rms, Ko, Do, rv, tv, newobj, sdi, sde, sdo, pv = r
    got = dict(rms=rms, K=Ko, D=Do.ravel(), rvecs=np.array(rv).reshape(-1, 3), tvecs=np.array(tv).reshape(-1, 3), std_int=sdi.ravel()[:9], std_ext=sde.reshape(-1, 6),
               pve=pv.ravel(), new_obj=None if newobj is None else newobj.reshape(-1, 3), std_obj=None if sdo is None else sdo.reshape(-1, 3))
    return got, st, r


def _same(r1, r2):
    for a, b in zip(r1, r2):
        if isinstance(a, tuple):
            if not all(np.array_equal(x, y) for x, y in zip(a, b)):
                return False
        elif a is None or b is None:
            if a is not b:
                return False
        elif np.asarray(a).tobytes() != np.asarray(b).tobytes():
            return False
    return True


def _assert_device_near_host(got, st, hs, tol=HOST_TOL):
    # The accept / reject sequences are not compared: once the run nears its minimum the trial costs differ from the previous one at
    # the rounding level, and which trial passes depends on how the reduced system was summed (measured on an H100: the sequences
    # part at the first rejected trial, after 7 to 10 kept ones).  The parameters both reach agree to HOST_TOL.
    assert st.n_steps >= 1 and len(hs["steps"]) >= 1
    worst = 0.0
    for k in ("rms", "std_int", "std_ext", "pve", "rvecs", "tvecs", "std_obj"):
        a, b = np.atleast_1d(np.asarray(got[k], np.float64)), np.atleast_1d(np.asarray(hs[k], np.float64))
        rel = np.abs(a - b) / np.maximum(np.abs(b), 1e-300)
        rel[(a == 0) & (b == 0)] = 0
        worst = max(worst, rel.max())
        assert rel.max() <= tol, (k, rel.max())
    rel_in = np.abs(cc.intrinsics(got) - cc.intrinsics(hs)) / np.maximum(np.abs(cc.intrinsics(hs)), 1e-300)
    assert rel_in.max() <= tol, rel_in
    d = np.abs(got["new_obj"].astype(np.float64) - hs["new_obj"].astype(np.float64))
    assert np.all(d <= tol * np.maximum(np.abs(hs["new_obj"]), 1e-3) + np.spacing(np.abs(hs["new_obj"]))), d.max()
    print("device vs host: largest relative difference %.3g" % max(worst, rel_in.max()))


CASES = [  # a subset of test_hostsim_calib_ro's sweep
    (2, 10, (6, 4), (1280, 720), "mild", 0, "n-2", (1.0, 1.004)),
    (4, 60, (5, 4), (3840, 2160), "pincushion", 0, "middle", (1.003, 0.998)),
    (5, 12, (16, 12), (1920, 1080), "mild", 0, "middle", (1.004, 1.0)),
    (7, 15, (7, 5), (1920, 1080), "mild", cv2.CALIB_ZERO_TANGENT_DIST | cv2.CALIB_FIX_PRINCIPAL_POINT, "middle", (1.004, 1.0)),
    (10, 15, (7, 5), (1920, 1080), "barrel", cv2.CALIB_USE_INTRINSIC_GUESS, "top-right", (1.004, 1.0)),
]


def _fixed(kind, grid):
    n = grid[0] * grid[1]
    return {"1": 1, "n-2": n - 2, "top-right": grid[0] - 1, "middle": n // 2 + grid[0] // 2}[kind]


@pytest.mark.parametrize("case", CASES, ids=[str(c[0]) for c in CASES])
def test_device_matches_host_and_cv2(case):
    seed, nv, grid, size, dist, flags, kind, scale = case
    O, I, K, D, true = rc.make_printed_problem(seed, nv, grid, size, dist, 0.2, scale)
    fixed = _fixed(kind, grid)
    Kg, Dg = (K * np.array([[1.01, 1, 1.003], [1, 0.99, 0.997], [1, 1, 1]]), D * 0.9) if flags & cv2.CALIB_USE_INTRINSIC_GUESS else (None, None)
    got, st, r1 = _device(O, I, size, fixed, Kg, Dg, flags)
    hs = rc.hs_calibrate_ro(O, I, size, fixed, Kg, Dg, flags)
    _assert_device_near_host(got, st, hs)
    ref = rc.cv2_calibrate_ro(O, I, size, fixed, Kg, Dg, flags)
    rc.assert_matches_cv2_ro(got, ref, O, fixed, "case %d" % seed)
    assert r1[5].shape == (1, grid[0] * grid[1], 3) and r1[5].dtype == np.float32 and r1[8].shape == (3 * grid[0] * grid[1], 1)
    _, st2, r2 = _device(O, I, size, fixed, Kg, Dg, flags)
    assert _same(r1, r2)
    assert st.n_evaluations >= 2 and st.device_ms > 0


def test_views_over_several_chunks_match_host():
    """600 views: the reduced system is streamed over chunks of 256, 256 and 88 views (CALIB_RO_CHUNK), in every step and in the
    final pass's per-view standard deviations."""
    O, I, K, D, true = rc.make_printed_problem(61, 600, (6, 4), (1920, 1080), "mild", 0.2, (1.004, 1.0))
    got, st, r1 = _device(O, I, (1920, 1080), 5)
    hs = rc.hs_calibrate_ro(O, I, (1920, 1080), 5)
    _assert_device_near_host(got, st, hs)
    _, _, r2 = _device(O, I, (1920, 1080), 5)
    assert _same(r1, r2)


def test_stored_cv2_result_of_a_large_board():
    """384 points x 30 views (m = 1 161): cv2's stored result (tests/golden/calib_ro_384x30.npz)."""
    O, I, size, fixed, ref = rc.golden()
    got, st, _ = _device(O, I, size, fixed)
    rc.assert_matches_cv2_ro(got, ref, O, fixed, "384 x 30")


def test_1024_points_1000_views_converges_and_is_deterministic():
    """The cap's board size (m = 3 081) over 1 000 views (4 chunks, the last of 232)."""
    O, I, K, D, true = rc.make_printed_problem(77, 1000, (32, 32), (3840, 2160), "mild", 0.2, (1.004, 1.0), square=0.01)
    fixed = 31
    got, st, r1 = _device(O, I, (3840, 2160), fixed)
    _, _, r2 = _device(O, I, (3840, 2160), fixed)
    assert _same(r1, r2)
    print("1024 x 1000: %.1f ms on the device, %d steps, %d launches, rms %.4f" % (st.device_ms, st.n_steps, st.kernel_launches, got["rms"]))
    assert got["rms"] < 0.3 and abs(got["K"][0, 0] / K[0, 0] - 1) < 1e-3
    assert np.all(got["std_obj"][1:fixed] > 0) and got["std_obj"][fixed].max() == 0
    assert np.all(np.isfinite(got["std_ext"])) and np.all(got["std_ext"] > 0)


def test_out_of_range_fixed_point_is_fid_calibrate_camera():
    O, I, K, D, true = rc.make_printed_problem(31, 8, (5, 4), (1280, 720), "mild", 0.2)
    st0 = _lib.fid_calib_stats()
    std = calib.calibrate_camera(O, I, (1280, 720), stats=st0)
    for fixed in (0, len(O[0]) - 1, -1):
        got, st, r = _device(O, I, (1280, 720), fixed)
        assert r[5] is None and r[8] is None
        assert _same(std, r[:5] + r[6:8] + r[9:])
        assert st.kernel_launches == st0.kernel_launches and bytes(st.steps) == bytes(st0.steps)


def test_refusals():
    O, I, K, D, true = rc.make_printed_problem(41, 6, (5, 4), (1280, 720), "mild", 0.2)

    def status(O, I, fixed=4, **kw):
        with pytest.raises(calib.CalibError) as e:
            calib.calibrate_camera_ro(O, I, (1280, 720), fixed, **kw)
        return e.value.calib_status

    assert status([O[0][:-1]] + O[1:], [I[0][:-1]] + I[1:]) == 7  # cv2: "... should be equal"
    moved = [o.copy() for o in O]
    moved[3][7, 0] += np.float32(1e-3)
    assert status(moved, I) == 7  # cv2: "... should be identical"
    assert status([true.astype(np.float32) for _ in O], I) == 2  # cv2: non-planar rig without a guess
    big = np.zeros((1025, 3), np.float32)
    big[:, 0], big[:, 1] = np.arange(1025) % 41, np.arange(1025) // 41
    assert status([big] * 2, [big[:, :2] * 10 + 5] * 2) == 1
    many = [big[:8]] * 4097
    assert status(many, [b[:, :2] * 10 + 5 for b in many]) == 6
    one = rc.make_printed_problem(51, 1, (5, 4), (1280, 720), "mild", 0.2)
    assert status(one[0], one[1]) == 9  # cv2: "There should be less vars to optimize ... than the number of residuals"


def _render_scaled(gray, board, R, t, K, sy, px_per_square=60):
    """charuco_oracle.render for a board printed sy times taller than its nominal geometry."""
    sx_, sy_ = board.getChessboardSize()
    sq = board.getSquareLength()
    margin = px_per_square // 2
    img = board.generateImage((sx_ * px_per_square + 2 * margin, sy_ * px_per_square + 2 * margin), marginSize=margin, borderBits=1)
    s = sq / px_per_square
    A = np.diag([1.0, sy, 1.0]) @ np.array([[s, 0, -margin * s], [0, s, -margin * s], [0, 0, 1]])
    Hm = np.asarray(K, np.float64) @ np.column_stack([R[:, 0], R[:, 1], t]) @ A
    H, W = gray.shape
    warped = cv2.warpPerspective(img, Hm, (W, H), flags=cv2.INTER_LINEAR)
    mask = cv2.warpPerspective(np.full_like(img, 255), Hm, (W, H), flags=cv2.INTER_NEAREST)
    gray[mask > 0] = warped[mask > 0]


def test_charuco_printed_taller_end_to_end():
    """Frames of a board printed 0.4 % taller than wide, through the batch ChArUco stage and charuco_views(complete=True), into the
    released calibration: it matches cv2 on the same corners, beats the standard calibration's rms and recovers the squares'
    aspect."""
    import charuco_oracle as co
    from fiducials_b200 import synth
    from fiducials_b200.board import charuco_board
    from fiducials_b200.node import Detector, default_params

    W, H = 1280, 720
    K, _ = synth.camera_for(W, H)
    board = charuco_board((7, 5), 0.04, 0.03)
    cvb = co.cv_board(board.size, board.square_length, board.marker_length, board.ids, board.legacy)
    rng = np.random.default_rng(9)
    frames = []
    for f in range(24):
        g = np.full((H, W), 128, np.uint8)
        R, t = co.board_pose_in_view(cvb, rng, K, W, H, kind=["near", "oblique"][f % 2])
        _render_scaled(g, cvb, R, t, K, 1.004)
        frames.append(cv2.cvtColor(co.blur_noise(g, rng), cv2.COLOR_GRAY2BGR))
    frames = np.ascontiguousarray(np.stack(frames))
    det = Detector(default_params(dictionary=co.DICT_ID), 0, W, H, len(frames))
    det.set_charuco_boards([board])
    det.detect_pose_batch(frames, K, np.zeros(5), 0.03)
    ch = det.last_charuco()
    det.close()
    O, I, kept = calib.charuco_views(board, [fr[0][1] for fr in ch], [fr[0][2] for fr in ch], complete=True)
    assert len(kept) >= 10 and all(np.array_equal(o, O[0]) for o in O)
    n = len(O[0])
    fixed = board.size[0] - 2  # the last corner of the first row: with corner 0 it pins the x extent
    got, st, r = _device(O, I, (W, H), fixed)
    ref = rc.cv2_calibrate_ro(O, I, (W, H), fixed)
    rc.assert_matches_cv2_ro(got, ref, O, fixed, "ChArUco")
    std = calib.calibrate_camera(O, I, (W, H))
    assert got["rms"] < std[0]
    new, nominal = got["new_obj"].astype(np.float64), O[0].astype(np.float64)
    aspect = (np.ptp(new[:, 1]) / np.ptp(new[:, 0])) / (np.ptp(nominal[:, 1]) / np.ptp(nominal[:, 0]))
    print("ChArUco printed 0.4 %% taller: %d views of %d corners, rms %.4f (standard %.4f), recovered aspect %.5f" % (len(O), n, got["rms"], std[0], aspect))
    assert abs(aspect - 1.004) < 2.5e-3  # 12 views of 24 corners pin it to about 2e-3 (cv2's own new points give the same figure)
