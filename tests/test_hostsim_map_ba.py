"""The host build of map_ba.cuh (fid_map_bundle_adjust's computation) against cv2 and scipy: the residuals and Jacobians against
cv2.projectPoints and central differences; the initial frame poses against cv2.aruco.Board + matchImagePoints + cv2.solvePnP; the
optimum against scipy.optimize.least_squares over a seeded sweep; the rules of which observations count; and the reported
standard deviations against the actual errors."""
import math

import cv2
import numpy as np
import pytest

import map_ba_cases as mc


def test_residual_and_jacobians_match_cv2_and_central_differences():
    rng = np.random.default_rng(5)
    for dist in (False, True):
        sc = mc.make_scene(3, n_markers=9, n_frames=12, walls=2, dist=dist, oblique=True)
        O = mc.object_points(sc)
        checked = 0
        for f in range(len(sc["counts"])):
            Rf, tf = sc["cams"][f]
            for j in range(sc["counts"][f]):
                i = list(sc["ids"]).index(sc["fids"][f, j])
                Rm = sc["R"][i] @ mc.rot(rng.normal(0, 0.05, 3))
                tm = sc["t"][i] + rng.normal(0, 0.01, 3)
                pf, pm = np.r_[Rf.ravel(), tf], np.r_[Rm.ravel(), tm]
                X = O[i] @ Rm.T + tm
                uv, J = cv2.projectPoints(X, cv2.Rodrigues(Rf)[0], tf, sc["K"], sc["D"])
                uv = uv.reshape(-1, 2)
                for k in range(4):
                    c = sc["corners"][f, j, k]
                    e, Jf, Jm = mc.hs_corner(O[i][k], c, sc["K"], sc["D"], pf, pm)
                    assert np.allclose(e, uv[k] - c.astype(np.float64), rtol=1e-9, atol=1e-9 * np.abs(uv[k]).max())
                    Jt = J[2 * k:2 * k + 2, 3:6]
                    assert np.allclose(Jf[:, 3:], Jt, rtol=1e-9, atol=1e-9 * np.abs(Jt).max())
                    assert np.allclose(Jm[:, 3:], Jt @ Rf, rtol=1e-9, atol=1e-9 * np.abs(Jt).max())
                    # the d/d theta columns: R Exp(delta), central differences
                    h = 1e-6
                    for col in range(3):
                        d = np.zeros(3)
                        d[col] = h
                        for which, J6 in ((0, Jf), (1, Jm)):
                            ep, em = [], []
                            for sgn, acc in ((1, ep), (-1, em)):
                                if which == 0:
                                    q = np.r_[(Rf @ mc.rot(sgn * d)).ravel(), tf]
                                    acc.append(mc.hs_corner(O[i][k], c, sc["K"], sc["D"], q, pm)[0])
                                else:
                                    q = np.r_[(Rm @ mc.rot(sgn * d)).ravel(), tm]
                                    acc.append(mc.hs_corner(O[i][k], c, sc["K"], sc["D"], pf, q)[0])
                            num = (ep[0] - em[0]) / (2 * h)
                            assert np.allclose(J6[:, col], num, rtol=1e-6, atol=1e-6 * np.abs(J6).max()), (which, col, J6[:, col], num)
                    checked += 1
        assert checked > 100


@pytest.mark.parametrize("walls,single", [(0, False), (3, False), (0, True)])
def test_initial_frame_poses_match_cv2_board_solvepnp(walls, single):
    """The initial pose is cv2's (Board + matchImagePoints + solvePnP on the float32 map corners) unless a marker's own pose
    composed with its map pose reprojects the frame's corners better than cv2's, or cv2's puts a corner behind the camera.  On a planar start map with
    several markers per frame that is every frame; single-marker frames keep whichever branch of the planar ambiguity
    reprojects better."""
    sc = mc.make_scene(11, n_markers=16, n_frames=30, walls=walls, visible=1 if single else 8, oblique=bool(walls), flat_start=True)
    g = mc.hs_bundle_adjust(sc, criteria="init")
    pos = {int(i): k for k, i in enumerate(sc["ids"])}
    O = mc.object_points(sc)
    same = other = 0
    for f in range(len(sc["counts"])):
        if g["status"][f] not in (1, 2):
            continue
        ok, rv, tv = mc.board_init_cv2(sc, f)
        assert ok
        # as rotation matrices: cv2 returns solvePnP's raw rvec, which may exceed pi; the call returns the wrapped one
        if np.allclose(cv2.Rodrigues(g["rvecs"][f])[0], cv2.Rodrigues(rv)[0], rtol=0, atol=1e-6) and \
                np.allclose(g["tvecs"][f], tv, rtol=0, atol=1e-6 * max(1.0, np.abs(tv).max())):
            same += 1
            continue
        ids = [int(v) for v in sc["fids"][f, :sc["counts"][f]]]
        obj = np.concatenate([(O[pos[i]] @ sc["start_R"][pos[i]].T + sc["start_t"][pos[i]]).astype(np.float32) for i in ids]).astype(np.float64)
        img = sc["corners"][f, :len(ids)].reshape(-1, 2).astype(np.float64)

        def err(r, t):
            return np.sum((cv2.projectPoints(obj, np.asarray(r, np.float64), np.asarray(t, np.float64), sc["K"], sc["D"])[0].reshape(-1, 2) - img) ** 2)

        R, t = cv2.Rodrigues(np.asarray(rv, np.float64))[0], np.asarray(tv, np.float64)
        behind = np.any((obj @ R.T + t)[:, 2] <= 0)  # cv2's pose has corners behind the camera: never taken
        assert behind or err(g["rvecs"][f], g["tvecs"][f]) < err(rv, tv), f
        other += 1
    assert same + other >= 10
    if not single:  # several markers: the board solve is the best candidate on (almost) every frame
        assert same >= 0.8 * (same + other), (same, other)


def _scipy_check(sc, **kw):
    g = mc.hs_bundle_adjust(sc, **kw)
    assert g["rc"] == 0, g["rc"]
    # scipy starts from the same initial frame poses
    i0 = mc.hs_bundle_adjust(sc, criteria="init")
    used = [f for f in range(len(sc["counts"])) if g["status"][f] == 1]
    ref = mc.scipy_bundle_adjust(sc, {f: mc.rot(i0["rvecs"][f]) for f in used}, {f: i0["tvecs"][f] for f in used})
    mc.assert_matches_scipy(g, ref)
    return g, ref


SWEEP = [  # (seed, markers, frames, walls, dist, noise, oblique, overrides, fixed)
    (1, 4, 10, 0, False, 0.0, False, False, 1),
    (2, 9, 30, 0, True, 0.5, False, False, 1),
    (3, 16, 40, 0, False, 1.0, True, True, 1),
    (4, 12, 40, 3, True, 0.3, True, False, 1),
    (5, 25, 60, 0, True, 0.5, False, True, 3),
    (6, 40, 100, 2, False, 0.5, True, False, 2),
    (7, 30, 150, 0, True, 0.5, True, False, 1),
]


@pytest.mark.parametrize("case", SWEEP, ids=[f"s{c[0]}-{c[1]}m-{c[2]}f" for c in SWEEP])
def test_optimum_matches_scipy(case):
    seed, nm, nf, walls, dist, noise, oblique, ov, nfix = case
    sc = mc.make_scene(seed, n_markers=nm, n_frames=nf, walls=walls, dist=dist, noise=noise, oblique=oblique, overrides=ov, n_fixed=nfix)
    g, ref = _scipy_check(sc)
    assert g["markers_used"] == len(ref["free"])
    if noise:
        assert g["final_rms"] < g["initial_rms"]


def test_disconnected_group_is_untouched_and_counted():
    a = mc.make_scene(21, n_markers=9, n_frames=30)
    b = mc.make_scene(22, n_markers=4, n_frames=8, n_fixed=0)
    sc = mc.join_disconnected(a, b)
    g = mc.hs_bundle_adjust(sc)
    assert g["rc"] == 0
    nb = len(b["ids"])
    assert g["markers_unreached"] == nb and g["frames_unreached"] == int(np.sum(b["counts"] > 0))
    assert np.all(g["status"][len(a["counts"]):][b["counts"] > 0] == 2)
    assert np.array_equal(g["R"][-nb:], sc["start_R"][-nb:]) and np.array_equal(g["t"][-nb:], sc["start_t"][-nb:])
    assert np.all(g["std"][-nb:] == 0)
    # the connected part is solved exactly as without the other group
    ga = mc.hs_bundle_adjust(a)
    assert np.array_equal(g["R"][:-nb], ga["R"]) and np.array_equal(g["t"][:-nb], ga["t"])


def test_duplicates_dropped_and_unmapped_ignored():
    sc = mc.make_scene(31, n_markers=9, n_frames=30)
    base = mc.hs_bundle_adjust(sc)
    s2 = dict(sc)
    s2["fids"], s2["corners"], s2["counts"] = sc["fids"].copy(), sc["corners"].copy(), sc["counts"].copy()
    # frame 3: an unmapped id appended; frame 5: one of its ids appended a second time (every observation of it there drops)
    f = 3
    s2["fids"][f, s2["counts"][f]] = 999
    s2["corners"][f, s2["counts"][f]] = s2["corners"][f, 0] + 3
    s2["counts"][f] += 1
    f = 5
    dup = s2["fids"][f, 0]
    s2["fids"][f, s2["counts"][f]] = dup
    s2["corners"][f, s2["counts"][f]] = s2["corners"][f, 0] + 2
    s2["counts"][f] += 1
    g = mc.hs_bundle_adjust(s2)
    assert g["dropped_unmapped"] == 1 and g["dropped_duplicate"] == 2
    assert g["observations"] == base["observations"] - 1
    # the same as dropping the duplicated id from frame 5 by hand
    s3 = dict(sc)
    s3["fids"], s3["corners"], s3["counts"] = sc["fids"].copy(), sc["corners"].copy(), sc["counts"].copy()
    n = s3["counts"][5]
    s3["fids"][5, :n - 1] = s3["fids"][5, 1:n]
    s3["corners"][5, :n - 1] = s3["corners"][5, 1:n]
    s3["fids"][5, n - 1] = -1
    s3["counts"][5] = n - 1
    g3 = mc.hs_bundle_adjust(s3)
    assert np.array_equal(g["R"], g3["R"]) and np.array_equal(g["t"], g3["t"])


def test_no_fixed_entry_is_refused():
    sc = mc.make_scene(41, n_markers=4, n_frames=10)
    g = mc.hs_bundle_adjust(sc, fixed=np.zeros(len(sc["ids"]), bool))
    assert g["rc"] == 2


def test_errors_fit_the_reported_uncertainty():
    """With 0.5 px noise the errors against the truth, over the standard deviations, have an RMS near 1 (the map frame is the
    fixed marker's: it sits at its true pose)."""
    z = []
    for seed in range(4):
        sc = mc.make_scene(100 + seed, n_markers=16, n_frames=60, noise=0.5, walls=2, oblique=True)
        g = mc.hs_bundle_adjust(sc)
        assert g["rc"] == 0
        for i in range(len(sc["ids"])):
            if sc["fixed"][i] or not np.all(g["std"][i] > 0):
                continue
            d = np.r_[mc.rot_delta(sc["R"][i], g["R"][i]), g["t"][i] - sc["t"][i]]
            z.extend(d / g["std"][i])
    z = np.array(z)
    r = math.sqrt(np.mean(z ** 2))
    assert 0.7 <= r <= 1.4, r


@pytest.mark.parametrize("height,tilt", [(0.05, 0.0), (0.03, 1.0), (0.0, 2.0), (0.08, 2.0)])
def test_a_fold_map_out_of_its_plane_is_improved(height, tilt):
    """A start map whose markers are off the ceiling's plane (heights and tilts, as a fold leaves them): solvePnP's non-planar DLT
    is poorly conditioned there, the single-marker candidates keep every frame's start near its pose, the run converges to the
    noise level and the map comes out closer to the truth than it went in."""
    sc = mc.make_scene(200, n_markers=25, n_frames=80, noise=0.5, perturb=(height, tilt))
    g = mc.hs_bundle_adjust(sc)
    assert g["rc"] == 0 and g["converged"] == 1 and g["init_failed"] == 0
    assert g["final_rms"] < 0.8, g["final_rms"]
    for f in range(len(sc["counts"])):
        if g["status"][f] == 1:
            Rf, tf = sc["cams"][f]
            # within the map's own error (centimetres); the mirror solution of a planar view is metres off
            assert np.linalg.norm(g["tvecs"][f] - tf) < 0.1 and np.linalg.norm(mc.rot_delta(Rf, mc.rot(g["rvecs"][f]))) < 0.05
    before = mc.map_error(sc, sc["start_R"], sc["start_t"])
    after = mc.map_error(sc, g["R"], g["t"])
    # positions start exact without a height error, rotations without tilt; the solve then leaves them at the noise level
    assert (after[0] < 0.5 * before[0] if height else after[0] < 0.05) and (after[1] < 0.5 * before[1] if tilt else after[1] < 0.02), (before, after)


def test_frames_that_see_only_fixed_entries():
    """No free marker (every observed entry fixed): the frames are still solved, and nothing in the map changes."""
    sc = mc.make_scene(61, n_markers=4, n_frames=12, n_fixed=4)
    g = mc.hs_bundle_adjust(sc)
    assert g["rc"] == 0 and g["markers_used"] == 0 and g["frames_used"] > 0 and g["converged"] == 1
    assert np.array_equal(g["R"], sc["start_R"]) and np.array_equal(g["t"], sc["start_t"]) and np.all(g["std"] == 0)
