"""Both planar pose hypotheses on the device (fid_pose_hypotheses, fid_set_pose_hypotheses / fid_last_pose_hypotheses) against
cv2.solvePnPGeneric(SOLVEPNP_IPPE_SQUARE), and the default outputs with the option on and off."""
import ctypes as C

import numpy as np
import pytest

from fiducials_b200 import _lib, synth
from fiducials_b200.node import MAXM, Detector, FiducialsNode, default_params
import ippe_oracle as io

pytestmark = pytest.mark.gpu

K_SYN, D_REF = synth.camera_for(640, 480)
D_ZERO = np.zeros(5)
FLEN = 0.14


def _host(det, cases, K, D, overrides=None):
    """fid_pose_hypotheses on (corners, len) cases; every case gets an id of its own whose override is its length."""
    ids = np.arange(len(cases), dtype=np.int32)
    corners = np.array([c for c, _ in cases], np.float32)
    ov = {int(i): float(L) for i, (_, L) in zip(ids, cases)} if overrides is None else overrides
    return [io.record_dict(r) for r in det.pose_hypotheses(ids, corners, K, D, FLEN, ov)], ids


def _check_host(det, cases, K, D):
    got, ids = _host(det, cases, K, D)
    for g, (c, L) in zip(got, cases):
        io.assert_matches(g, io.pose_hypotheses(c, K, D, L))


@pytest.fixture(scope="module")
def det640():
    d = Detector(default_params(dictionary=synth.CONFIGS["C1"][3]), 0, 640, 480, 2)
    yield d
    d.close()


@pytest.mark.parametrize("name", ["tag01", "tag245", "img403", "bag"])
def test_host_corners_golden(kat, det640, name):
    L = float(np.float32(float(kat[name + "_len"])))
    _check_host(det640, [(c, L) for c in kat[name + "_corners"]], kat[name + "_K"].reshape(3, 3), kat[name + "_D"])


@pytest.mark.parametrize("D", [D_REF, D_ZERO], ids=["D_ref", "D_zero"])
@pytest.mark.parametrize("kind,seed", [("far", 1), ("far", 2), ("tilted", 3), ("mixed", 4)])
def test_host_corners_synthetic(det640, kind, seed, D):
    _check_host(det640, io.synthetic_cases(seed, K_SYN, D, kind=kind), K_SYN, D)


def test_host_corners_default_length_and_overrides(det640):
    cases = io.synthetic_cases(7, K_SYN, D_REF, kind="mixed", n=24)
    ids = np.arange(24, dtype=np.int32)
    overrides = {1: 0.05, 5: 0.2, 9: 0.3333}  # the others take fiducial_len, narrowed to float
    lens = [overrides.get(i, float(np.float32(FLEN))) for i in range(24)]
    got = det640.pose_hypotheses(ids, np.array([c for c, _ in cases]), K_SYN, D_REF, FLEN, overrides)
    for r, (c, _), L, i in zip(got, cases, lens, ids):
        assert r.fiducial_id == i
        io.assert_matches(io.record_dict(r), io.pose_hypotheses(c, K_SYN, D_REF, L))


@pytest.mark.parametrize("D", [D_REF, D_ZERO], ids=["D_ref", "D_zero"])
def test_host_corners_iterative_in_second_basin(det640, D):
    c, L, ref = io.iterative_in_second_basin(K_SYN, D)
    (got,), _ = _host(det640, [(c, L)], K_SYN, D)
    swapped = io.assert_matches(got, ref)
    assert ref["iterative_match"] == 1 and got["iterative_match"] == (0 if swapped else 1)


def test_host_corners_degenerate(det640):
    quads = [(np.full((4, 2), 300.0, np.float32), FLEN), (np.array([[300, 200], [310, 200], [320, 200], [330, 200]], np.float32), FLEN)]
    got, _ = _host(det640, quads, K_SYN, D_ZERO)
    for g in got:
        assert g["n"] == 0 and g["iterative_match"] == -1
        for k in ("rvec", "tvec", "rms"):
            assert np.all(np.isfinite(g[k])) and not np.any(g[k])


def _frames(cfg, seeds, blank=()):
    fr = []
    for i, s in enumerate(seeds):
        bgr, _, K, D, d = synth.make_config_frame(cfg, s)
        fr.append(np.full_like(bgr, 128) if i in blank else bgr)
    return np.ascontiguousarray(np.stack(fr)), K, D, d


def _check_batch(det, out, hyps, K, D):
    counts, ids, corners, tfs = out
    n_markers = 0
    for f in range(len(counts)):
        for m in range(int(counts[f])):
            r = hyps[f * MAXM + m]
            t = tfs[f * MAXM + m]
            assert r.fiducial_id == ids[f, m] == t.fiducial_id
            ref = io.pose_hypotheses(corners[f, m], K, D, float(np.float32(FLEN)))  # the oracle on the device's own corners
            if ref["n"]:
                ref["iterative_match"] = io._closer(np.array(t.rvec), ref["rvec"])  # the basin of the device's ITERATIVE pose
            io.assert_matches(io.record_dict(r), ref, "frame %d marker %d" % (f, m))
            n_markers += 1
    return n_markers


@pytest.mark.parametrize("cfg,seeds,blank,max_batch", [("C1", range(7), (2, 5), 2), ("C2", range(4), (), 2)])
def test_batch_path(cfg, seeds, blank, max_batch):
    """submit/collect with the option on: batches of several chunks (max_batch 2), frames without markers, every record against
    the oracle on the device's corners."""
    frames, K, D, d = _frames(cfg, seeds, blank)
    W, H = frames.shape[2], frames.shape[1]
    det = Detector(default_params(dictionary=d), 0, W, H, max_batch)
    det.set_pose_hypotheses(True)
    half = len(frames) // 2
    a, b = np.ascontiguousarray(frames[:half]), np.ascontiguousarray(frames[half:])
    det.submit_batch(a, K, D, FLEN)
    det.submit_batch(b, K, D, FLEN)  # two batches in flight: each keeps its own records
    n, counts = 0, []
    for part in (a, b):
        out = det.collect_batch()
        hyps = det.last_pose_hypotheses()
        assert len(hyps) == len(part) * MAXM
        n += _check_batch(det, out, hyps, K, D)
        counts += out[0].tolist()
    assert all(counts[f] == 0 for f in blank) and n == sum(counts)
    assert n >= (4 if cfg == "C1" else 16) * (len(frames) - len(blank)) * 0.9
    # the synchronous batch call fills the same records
    out = det.detect_pose_batch(frames, K, D, FLEN)
    _check_batch(det, out, det.last_pose_hypotheses(), K, D)
    det.close()


def test_default_outputs_unchanged_by_the_option():
    frames, K, D, d = _frames("C2", [11, 12, 13])
    W, H = frames.shape[2], frames.shape[1]
    det = Detector(default_params(dictionary=d), 0, W, H, 2)
    res = {}
    for on in (False, True, False):
        det.set_pose_hypotheses(on)
        det.submit_batch(frames, K, D, FLEN)
        counts, ids, corners, tfs = det.collect_batch()
        res.setdefault(on, []).append((counts.tobytes(), ids.tobytes(), corners.tobytes(), bytes(tfs)))
    assert res[False][0] == res[True][0] == res[False][1]
    det.close()


def test_errors():
    frames, K, D, d = _frames("C1", [0, 1])
    det = Detector(default_params(dictionary=d), 0, 640, 480, 2)
    lib, nf = det.lib, C.c_int(0)
    buf = (_lib.fid_pose_hypotheses * (2 * MAXM))()
    # option off for the batch -> FID_ERR_INVALID_ARG
    det.submit_batch(frames, K, D, FLEN)
    det.collect_batch()
    assert lib.fid_last_pose_hypotheses(det.h, MAXM, C.byref(nf), C.cast(buf, C.c_void_p)) == -1
    # not while a batch is in flight
    det.submit_batch(frames, K, D, FLEN)
    assert lib.fid_set_pose_hypotheses(det.h, 1) == -1
    det.collect_batch()
    _lib.check(lib.fid_set_pose_hypotheses(det.h, 1))
    # on, but without a camera: no pose, no records
    det.submit_batch(frames)
    det.collect_batch()
    assert lib.fid_last_pose_hypotheses(det.h, MAXM, C.byref(nf), C.cast(buf, C.c_void_p)) == -1
    det.submit_batch(frames, K, D, FLEN)
    counts = det.collect_batch()[0]
    assert counts.max() >= 2
    assert lib.fid_last_pose_hypotheses(det.h, int(counts.max()) - 1, C.byref(nf), C.cast(buf, C.c_void_p)) == -5  # FID_ERR_CAPACITY
    assert lib.fid_last_pose_hypotheses(det.h, int(counts.max()), C.byref(nf), C.cast(buf, C.c_void_p)) == 0 and nf.value == 2
    assert lib.fid_set_pose_hypotheses(det.h, 0) == 0
    det.close()


def test_node_attaches_records_by_id():
    bgr, _, K, D, d = synth.make_config_frame("C1", 3)
    plain = FiducialsNode(dictionary=d, fiducial_len=FLEN, max_width=640, max_height=480, max_batch=2)
    node = FiducialsNode(dictionary=d, fiducial_len=FLEN, max_width=640, max_height=480, max_batch=2, pose_hypotheses=True)
    for n in (plain, node):
        n.camInfoCallback(K, D, "camera")
    fta0 = plain.poseEstimateCallback(plain.imageCallback(bgr))
    fta = node.poseEstimateCallback(node.imageCallback(bgr))
    assert fta.transforms == fta0.transforms and not hasattr(fta0, "pose_hypotheses")
    assert set(fta.pose_hypotheses) == set(t.fiducial_id for t in fta.transforms) and len(fta.transforms) >= 3
    for f in node.imageCallback(bgr).fiducials:
        c = np.array([f.x0, f.y0, f.x1, f.y1, f.x2, f.y2, f.x3, f.y3], np.float32).reshape(4, 2)
        io.assert_matches(io.record_dict(fta.pose_hypotheses[f.fiducial_id]), io.pose_hypotheses(c, K, D, float(np.float32(FLEN))))
    frames = np.ascontiguousarray(np.stack([bgr, bgr, bgr]))
    batch0, batch = plain.process_batch(frames), node.process_batch(frames)
    for a, b in zip(batch0, batch):  # the batch path (k_pose_hypotheses after k_finish) gives the records of the host-corner call
        assert a.transforms == b.transforms and set(b.pose_hypotheses) == set(fta.pose_hypotheses)
        for k, v in b.pose_hypotheses.items():
            g, r = io.record_dict(v), io.record_dict(fta.pose_hypotheses[k])
            assert g["iterative_match"] == r["iterative_match"] and np.abs(g["rvec"] - r["rvec"]).max() < 1e-9 and np.abs(g["tvec"] - r["tvec"]).max() < 1e-9
