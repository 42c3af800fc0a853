"""The per-marker pose on the device over the seeded geometry classes of tests/pose_sweep_cases.py: fid_pose (k_pose) against
cv2.solvePnP and against the host build of the same source, rendered frames through the batch path (k_finish) against cv2 on the
device's own corners and against fid_pose, and the ITERATIVE basin fid_pose_hypotheses reports on half-turn markers."""
import math

import cv2
import numpy as np
import pytest

from fiducials_b200 import synth
from fiducials_b200.node import MAXM, Detector, default_params
import hostsim_util as hs
import ippe_oracle as io
import pose_sweep_cases as ps

pytestmark = pytest.mark.gpu

N = 700
CALL_SIZES = (1, 63, 64, 65, 507)  # k_pose runs 64-thread blocks: partial blocks, one exact block, several blocks
SEEDS = {c: 9300 + i for i, c in enumerate(ps.CLASSES)}
DEVICE_HOST_TOL = 1e-7


@pytest.fixture(scope="module")
def det():
    d = Detector(default_params(dictionary=synth.CONFIGS["C1"][3]), 0, 640, 480, 2)
    yield d
    d.close()


def record(t):
    return dict(rvec=np.array(t.rvec[:]), tvec=np.array(t.translation[:]), quat=np.array(t.rotation[:]), image_error=t.image_error, object_error=t.object_error,
                area=t.fiducial_area, lm_iters=int(t.reserved))


def device_poses(det, cs, K, D, sizes=CALL_SIZES):
    """fid_pose over the cases, in calls of the given sizes (the rest in one more call)."""
    out, i = [], 0
    for n in list(sizes) + [len(cs)]:
        part = cs[i : i + n] if n < len(cs) else cs[i:]
        if not part:
            break
        ids = np.array([c.marker_id for c in part], np.int32)
        tfs = det.pose(ids, np.array([c.corners for c in part]), K, D, ps.FLEN, ps.OVERRIDES)
        assert [t.fiducial_id for t in tfs] == ids.tolist()
        out += [record(t) for t in tfs]
        i += len(part)
    assert len(out) == len(cs)
    return out


def host_poses(cs, K, D):
    o = hs.pose(np.array([c.corners for c in cs]), K, D, np.array([c.length for c in cs], np.float32), ps.FLEN)
    return [dict(rvec=r[0:3], tvec=r[3:6], lm_iters=int(r[13])) for r in o]


@pytest.mark.parametrize("cls", ps.CLASSES)
def test_fid_pose_matches_cv2_and_the_host_build(det, cls):
    K, D, W, H = ps.CAMERAS[cls]
    cs = ps.cases(cls, SEEDS[cls], N)
    got = device_poses(det, cs, K, D)
    host = host_poses(cs, K, D)
    ties, worst = 0, 0.0
    for c, g, h in zip(cs, got, host):
        d = ps.compare(g, ps.oracle(c.corners, K, D, c.length), c, K, D)
        ps.check(d, c.name)
        ties += d["half_turn_tie"]
        # the same source built for the host: the same LM run (finding 3 -- a miscompile moves a pose or its iteration count).
        # The last accepted step may still differ by up to the stop test's size (finding 12): measured <= 4.4e-8.
        assert g["lm_iters"] == h["lm_iters"], (c.name, g["lm_iters"], h["lm_iters"])
        dh = max(np.abs(g["rvec"] - h["rvec"]).max(), np.abs(g["tvec"] - h["tvec"]).max())
        assert dh <= (DEVICE_HOST_TOL if g["lm_iters"] < ps.LM_CAP else ps.TOL), (c.name, dh)
        worst = max(worst, dh)
    print("\n%s: device vs host build max %.3g" % (cls, worst))
    assert ties <= (2 if cls.startswith("half_turn") else 0), (cls, ties)


def test_fid_pose_4096_markers_in_one_call(det):
    K, D, W, H = ps.CAMERAS["mixed"]
    cs = ps.cases("mixed", 9399, 4096)
    got = device_poses(det, cs, K, D, sizes=(4096,))
    host = host_poses(cs, K, D)
    for c, g, h in zip(cs, got, host):
        ps.check(ps.compare(g, ps.oracle(c.corners, K, D, c.length), c, K, D), c.name)
        assert g["lm_iters"] == h["lm_iters"], c.name


# ---- rendered frames through the batch path ---------------------------------------------------------------------------------
DICT = 10


def _axis_aligned_frame(seed):
    """Markers from generateImageMarker pasted without rotation on a flat background: fronto-parallel, zero spin."""
    d = cv2.aruco.getPredefinedDictionary(DICT)
    rng = np.random.default_rng(seed)
    img = np.full((480, 640), 205, np.uint8)
    for k in range(4):
        side = int(rng.integers(70, 120))
        y0, x0 = 30 + 230 * (k // 2) + int(rng.integers(0, 60)), 40 + 300 * (k % 2) + int(rng.integers(0, 100))
        img[y0 : y0 + side, x0 : x0 + side] = cv2.aruco.generateImageMarker(d, int(rng.integers(0, 250)), side)
    img = cv2.GaussianBlur(img, (0, 0), 0.8)
    return np.repeat(img[:, :, None], 3, axis=2)


def _frames():
    axis = [_axis_aligned_frame(s) for s in range(4)]
    steep = [synth.make_frame(640, 480, 4, DICT, seed=s, max_tilt_deg=72.0)[0] for s in range(6)]
    return np.ascontiguousarray(np.stack(axis + steep))


@pytest.mark.parametrize("D", [synth.camera_for(640, 480)[1], np.zeros(5)], ids=["D_ref", "D_zero"])
def test_batch_path_rendered_frames(D):
    K = synth.camera_for(640, 480)[0]
    frames = _frames()
    det = Detector(default_params(dictionary=DICT), 0, 640, 480, 4)
    try:
        counts, ids, corners, tfs = det.detect_pose_batch(frames, K, D, ps.FLEN)
        counts, ids, corners = counts.copy(), ids.copy(), corners.copy()
        recs = [[tfs[f * MAXM + m] for m in range(int(counts[f]))] for f in range(len(frames))]
        n = 0
        for f in range(len(frames)):
            nf = int(counts[f])
            assert nf >= 3, (f, nf)
            single = det.pose(ids[f, :nf], corners[f, :nf], K, D, ps.FLEN)  # k_pose on k_finish's corners
            for m in range(nf):
                t = recs[f][m]
                assert bytes(t) == bytes(single[m]), ("frame %d marker %d: k_finish and fid_pose differ" % (f, m))
                c = ps.Case("frame", f, m, corners[f, m], 0, float(np.float32(ps.FLEN)))
                ps.check(ps.compare(record(t), ps.oracle(corners[f, m], K, D, c.length), c, K, D), c.name)
                n += 1
        assert n >= 30
    finally:
        det.close()


def test_pose_hypotheses_basin_on_half_turns(det):
    """fid_pose_hypotheses' iterative_match names the IPPE solution closer to the published (ITERATIVE) pose; on half-turn markers
    it must agree with both fid_pose's rvec and cv2's.  (The IPPE solutions themselves are not compared with cv2 here: at an exact
    half turn cv2's IPPE_SQUARE can return a rotation 0.15 rad off, with a reprojection RMS 1e4 times ours -- finding 12.)"""
    K, D, W, H = ps.CAMERAS["half_turn"]
    cs = ps.cases("half_turn", 9398, 300)
    ids = np.array([c.marker_id for c in cs], np.int32)
    corners = np.array([c.corners for c in cs])
    hyps = det.pose_hypotheses(ids, corners, K, D, ps.FLEN, ps.OVERRIDES)
    poses = device_poses(det, cs, K, D, sizes=())
    n2 = n_distinct = 0
    for c, r, p in zip(cs, hyps, poses):
        got = io.record_dict(r)
        if got["n"] != 2:
            continue
        n2 += 1
        # unless the two solutions are the same rotation to 1e-5 (fronto-parallel: then "closer" is a tie that a 1e-8 difference
        # decides), fid_pose's rvec and cv2's pick the solution the record names
        if np.abs(ps.rotation_matrix(got["rvec"][0]) - ps.rotation_matrix(got["rvec"][1])).max() > 1e-5:
            ref = ps.oracle(c.corners, K, D, c.length)
            assert got["iterative_match"] == io._closer(p["rvec"], got["rvec"]), c.name
            assert got["iterative_match"] == io._closer(ref["rvec"], got["rvec"]), c.name
            n_distinct += 1
    print("\nhalf-turn markers with two solutions: %d, of them distinguishable: %d" % (n2, n_distinct))
    assert n2 >= 250 and n_distinct >= 250, (n2, n_distinct)
