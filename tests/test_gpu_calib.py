"""fid_calibrate_camera on the device against the host build of calib.cuh (same iterations, same accept / reject sequence, the
same numbers) and against cv2.calibrateCameraExtended, at sizes up to 4 000 views, and end to end from rendered ChArUco frames
through the batch detector and charuco_views."""
import cv2
import numpy as np
import pytest

import calib_cases as cc
from fiducials_b200 import _lib, calib

pytestmark = pytest.mark.gpu


def _device(O, I, size, K=None, D=None, flags=0, criteria=None):
    st = _lib.fid_calib_stats()
    r = calib.calibrate_camera(O, I, size, K, D, flags, criteria, stats=st)
    rms, Ko, Do, rv, tv, sdi, sde, pv = r
    got = dict(rms=rms, K=Ko, D=Do.ravel(), rvecs=np.array(rv).reshape(-1, 3), tvecs=np.array(tv).reshape(-1, 3), std_int=sdi.ravel()[:9], std_ext=sde.reshape(-1, 6),
               pve=pv.ravel())
    return got, st, r


def _assert_device_equals_host(got, st, hs, tol=1e-10):
    assert st.n_steps == len(hs["steps"]) and bytes(st.steps[: st.n_steps]) == hs["steps"].tobytes()
    for k in ("rms", "std_int", "std_ext", "pve", "rvecs", "tvecs"):
        a, b = np.asarray(got[k], np.float64), np.asarray(hs[k], np.float64)
        assert np.all(np.abs(a - b) <= tol * np.maximum(np.abs(b), 1e-300)), (k, np.abs(a - b).max())
    assert np.all(np.abs(cc.intrinsics(got) - cc.intrinsics(hs)) <= tol * np.abs(cc.intrinsics(hs)))


CASES = [
    (101, 3, (6, 4), (640, 480), "zero", 0.0, 0.0, 0, None),
    (102, 25, (6, 4), (1920, 1080), "mild", 0.1, 0.4, 0, None),
    (103, 60, (11, 8), (3840, 2160), "barrel", 0.3, 0.5, 0, None),
    (104, 12, (32, 32), (1920, 1080), "pincushion", 0.2, 0.3, 0, None),
    (105, 20, (6, 4), (1280, 720), "mild", 0.2, 0.3, cv2.CALIB_FIX_ASPECT_RATIO | cv2.CALIB_ZERO_TANGENT_DIST | cv2.CALIB_FIX_K3, None),
    (106, 20, (6, 4), (1920, 1080), "barrel", 0.2, 0.3, cv2.CALIB_USE_INTRINSIC_GUESS | cv2.CALIB_FIX_PRINCIPAL_POINT, None),
    (107, 20, (6, 4), (1920, 1080), "mild", 0.2, 0.3, 0, (cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS, 100, 1e-12)),
]


@pytest.mark.parametrize("case", CASES, ids=[str(c[0]) for c in CASES])
def test_device_matches_host_and_cv2(case):
    seed, nv, grid, size, dist, noise, partial, flags, crit = case
    O, I, K, D = cc.make_problem(seed, nv, grid, size, dist, noise, partial)
    Kg, Dg = (K, D * 0.9) if flags & cv2.CALIB_USE_INTRINSIC_GUESS else (K if flags & cv2.CALIB_FIX_ASPECT_RATIO else None, None)
    got, st, r1 = _device(O, I, size, Kg, Dg, flags, crit)
    hs = cc.hs_calibrate(O, I, size, Kg, Dg, flags, crit)
    _assert_device_equals_host(got, st, hs)
    ref, converged = cc.cv2_converged(O, I, size, Kg, Dg, flags, crit)
    assert converged
    cc.assert_matches_cv2(got, ref, "case %d" % seed)
    # a second run of the same input: the same bits
    _, st2, r2 = _device(O, I, size, Kg, Dg, flags, crit)
    assert r1[0] == r2[0] and all(np.array_equal(np.asarray(a), np.asarray(b)) for a, b in zip(r1[1:], r2[1:]))
    assert st.n_evaluations >= 2 and st.device_ms > 0


@pytest.mark.parametrize("nv", [1000, 4000])
def test_large_problems_match_host(nv):
    O, I, K, D = cc.make_problem(200 + nv, nv, (6, 4), (1920, 1080), "mild", 0.2, 0.3)
    got, st, _ = _device(O, I, (1920, 1080))
    hs = cc.hs_calibrate(O, I, (1920, 1080))
    _assert_device_equals_host(got, st, hs)
    assert abs(got["K"][0, 0] / K[0, 0] - 1) < 1e-2


def test_errors_and_unsupported_flags():
    O, I, K, D = cc.make_problem(300, 5, (6, 4), (1920, 1080), "mild", 0.1)
    Oc, Ic = list(O), list(I)
    Oc[1], Ic[1] = O[1][:6], I[1][:6]  # one grid row: no homography, as in cv2
    with pytest.raises(calib.CalibError) as e:
        calib.calibrate_camera(Oc, Ic, (1920, 1080))
    assert e.value.calib_status == 3
    with pytest.raises(_lib.FidError) as e:
        calib.calibrate_camera(O, I, (1920, 1080), flags=cv2.CALIB_RATIONAL_MODEL)
    assert e.value.status == -4
    # one view: accepted, like cv2
    got, st, _ = _device(O[:1], I[:1], (1920, 1080))
    hs = cc.hs_calibrate(O[:1], I[:1], (1920, 1080))
    assert st.n_steps == len(hs["steps"]) and abs(got["rms"] - hs["rms"]) <= 1e-10 * max(hs["rms"], 1e-12)


def test_charuco_frames_end_to_end():
    """Rendered ChArUco frames through a batch with the board set, the corners through charuco_views, into the device and cv2."""
    import charuco_oracle as co
    from fiducials_b200 import synth
    from fiducials_b200.board import charuco_board
    from fiducials_b200.node import Detector, default_params

    W, H = 1280, 720
    K, _ = synth.camera_for(W, H)
    board = charuco_board((7, 5), 0.04, 0.03)
    cvb = co.cv_board(board.size, board.square_length, board.marker_length, board.ids, board.legacy)
    rng = np.random.default_rng(5)
    frames = []
    for f in range(16):
        g = np.full((H, W), 128, np.uint8)
        R, t = co.board_pose_in_view(cvb, rng, K, W, H, kind=["near", "oblique"][f % 2])
        co.render(g, cvb, R, t, K)
        frames.append(cv2.cvtColor(co.blur_noise(g, rng), cv2.COLOR_GRAY2BGR))
    frames = np.ascontiguousarray(np.stack(frames))
    det = Detector(default_params(dictionary=co.DICT_ID), 0, W, H, 4)
    det.set_charuco_boards([board])
    det.detect_pose_batch(frames, K, np.zeros(5), 0.03)
    ch = det.last_charuco()
    det.close()
    O, I, kept = calib.charuco_views(board, [fr[0][1] for fr in ch], [fr[0][2] for fr in ch])
    assert len(kept) >= 10
    got, st, _ = _device(O, I, (W, H))
    hs = cc.hs_calibrate(O, I, (W, H))
    _assert_device_equals_host(got, st, hs)
    ref = cc.cv2_calibrate(O, I, (W, H))
    assert abs(got["rms"] / ref["rms"] - 1) <= 1e-6
    assert np.abs(cc.intrinsics(got) - cc.intrinsics(ref)).max() <= 1e-3 * np.abs(cc.intrinsics(ref)).max()
