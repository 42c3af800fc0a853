"""GPU parity tests proper: the CUDA path through the C-ABI vs the cv2 oracle on the same seeded
inputs, the committed reference goldens, edge cases, and size-independent properties at
BASELINE.json's full sizes.  Tolerances (BASELINE.md section 4): ids identical and in identical
order; corners within 1e-3 px; rvec/tvec within 1e-3; image/object error and area within 1e-6
relative; integer stages (gray, threshold planes, quad candidates) bit-exact."""
import ctypes as C
import math

import numpy as np
import pytest

from fiducials_b200 import synth
from oracle import aruco_oracle as ao

pytestmark = pytest.mark.gpu

# aruco_detect/test/aruco_images_test.cpp:96-109, 125-147
GOLD = {
    "tag01": {1: [569.89917, 201.55890, 777.42560, 206.85025, 767.95856, 415.37830, 565.75311, 409.24496]},
    "tag245": {
        245: [307.68246, 157.38346, 545.10131, 167.04420, 540.11614, 403.27578, 305.64746, 395.01422],
        246: [671.51892, 173.46070, 900.29650, 178.44973, 895.06933, 407.39855, 666.39910, 403.12911],
    },
}


@pytest.fixture(scope="module")
def det_cache():
    from fiducials_b200.node import Detector, default_params

    cache = {}

    def get(dict_id, W, H, batch=1):
        key = (dict_id, W, H, batch)
        if key not in cache:
            cache[key] = Detector(default_params(dictionary=dict_id), 0, W, H, batch)
        return cache[key]

    yield get
    for d in cache.values():
        d.close()


def _check_detect(det, bgr, dict_id):
    ids, corners = det.detect(bgr)
    rids, rcorners = ao.detect(bgr, dict_id)
    assert ids.tolist() == rids.tolist()
    if len(ids):
        assert np.abs(corners - rcorners).max() <= 1e-3
    return ids, corners


# ---- integer stages: bit exact ------------------------------------------------------------------
@pytest.mark.parametrize("case", ["C1", "noise", "odd", "flat", "kat"])
def test_threshold_planes_bit_exact(det_cache, kat, case):
    rng = np.random.default_rng(11)
    if case == "C1":
        bgr = synth.make_config_frame("C1", 0)[0]
    elif case == "noise":
        bgr = rng.integers(0, 256, (240, 352, 3), dtype=np.uint8)
    elif case == "odd":
        bgr = rng.integers(0, 256, (131, 203, 3), dtype=np.uint8)  # not a multiple of the tile or of 32
    elif case == "flat":
        bgr = np.full((96, 160, 3), 200, np.uint8)
    else:
        bgr = kat.frame("tag01")
    H, W = bgr.shape[:2]
    det = det_cache(7, max(W, 16), max(H, 16))
    g, planes = det.debug_threshold(bgr)
    rg = ao.gray(bgr)
    assert np.array_equal(g, rg)
    rp = ao.threshold_planes(rg)
    assert planes.shape == rp.shape
    assert np.array_equal(planes, rp), [int((planes[s] != rp[s]).sum()) for s in range(len(rp))]


@pytest.mark.parametrize("cfg,seed", [("C1", 0), ("C1", 4), ("C3", 1)])
def test_quad_candidates_bit_exact(det_cache, cfg, seed):
    bgr, _, K, D, d = synth.make_config_frame(cfg, seed)
    H, W = bgr.shape[:2]
    det = det_cache(d, W, H)
    det.detect(bgr)
    quads, scale, clen = det.debug_candidates()
    ref = ao.quad_candidates(ao.gray(bgr))
    assert len(quads) == len(ref) and len(ref) > 10
    for i, (s, q, n) in enumerate(ref):
        assert s == scale[i] and n == clen[i] and np.array_equal(q, quads[i])


# ---- detect + pose vs oracle --------------------------------------------------------------------
@pytest.mark.parametrize("cfg,seed", [("C1", 0), ("C1", 1), ("C1", 2), ("C1", 3), ("C3", 0), ("C3", 7), ("C2", 0), ("C2", 5)])
def test_detect_pose_matches_oracle(det_cache, cfg, seed):
    bgr, truth, K, D, d = synth.make_config_frame(cfg, seed)
    H, W = bgr.shape[:2]
    det = det_cache(d, W, H)
    ids, corners = _check_detect(det, bgr, d)
    tid = sorted(m for m, _ in truth)  # every synthetic marker found, except ones cut by the frame edge (cv2 drops those too)
    assert set(ids.tolist()) <= set(tid) and len(ids) >= len(tid) - 1
    rids, rcorners, rvecs, tvecs, fields = ao.detect_and_pose(bgr, d, K, D, 0.14)
    tfs = det.pose(ids, corners, K, D, 0.14)
    for i, t in enumerate(tfs):
        assert t.fiducial_id == int(rids[i])
        assert np.abs(np.array(t.rvec) - rvecs[i]).max() < 1e-3
        assert np.abs(np.array(t.translation) - tvecs[i]).max() < 1e-3
        assert np.abs(np.array(t.rotation) - fields[i]["rotation"]).max() < 1e-3
    # same corners in -> errors/areas agree to 1e-6 relative (fed with the oracle's corners)
    tfs = det.pose(rids, rcorners, K, D, 0.14)
    for i, t in enumerate(tfs):
        f = fields[i]
        assert abs(t.image_error - f["image_error"]) <= 1e-6 * max(1.0, f["image_error"]) + 1e-7
        assert abs(t.object_error - f["object_error"]) <= 1e-6 * max(1e-3, f["object_error"]) + 1e-9
        assert abs(t.fiducial_area - f["fiducial_area"]) <= 1e-6 * f["fiducial_area"]


@pytest.mark.parametrize("name", ["tag01", "tag245", "img403", "bag"])
def test_reference_fixture_frames(det_cache, kat, name):
    bgr = kat.frame(name)
    det = det_cache(7, 1280, 960)
    ids, corners = det.detect(bgr)
    assert ids.tolist() == kat[name + "_ids"].tolist()
    assert np.abs(corners - kat[name + "_corners"]).max() <= 1e-3
    if name in GOLD:  # the reference's own golden corners
        for i, fid in enumerate(ids.tolist()):
            assert np.abs(corners[i].reshape(-1) - np.array(GOLD[name][fid], np.float32)).max() < 1.3e-4 + 1e-3
    flen = float(kat[name + "_len"])
    tfs = det.pose(ids, corners, kat[name + "_K"], kat[name + "_D"], flen)
    for i, t in enumerate(tfs):
        assert np.abs(np.array(t.rvec) - kat[name + "_rvecs"][i]).max() < 1e-3
        assert np.abs(np.array(t.translation) - kat[name + "_tvecs"][i]).max() < 1e-3
        assert np.abs(np.array(t.rotation) - kat[name + "_quat"][i]).max() < 1e-3
        e = kat[name + "_errs"][i]
        assert abs(t.fiducial_area / e[2] - 1) < 1e-4


def test_bag_pair_through_gpu(det_cache, kat):
    """image bag -> GPU detect+pose must reproduce the reference's golden FiducialTransformArray."""
    det = det_cache(7, 1280, 960)
    ids, corners = det.detect(kat.frame("bag"))
    tfs = {t.fiducial_id: t for t in det.pose(ids, corners, kat["bag_K"], kat["bag_D"], 0.14)}
    for j, fid in enumerate(kat["bag_golden_ids"].tolist()):
        t = tfs[fid]
        assert np.abs(np.array(t.translation) - kat["bag_golden_t"][j]).max() < 1e-4
        q, gq = np.array(t.rotation), kat["bag_golden_q"][j]
        assert min(np.abs(q - gq).max(), np.abs(q + gq).max()) < 1e-4


def test_node_mirror_messages(kat):
    from fiducials_b200.node import FiducialsNode

    node = FiducialsNode(dictionary=7, fiducial_len=0.145, max_width=1280, max_height=960, ignore_fiducials=[246])
    node.camInfoCallback(kat["tag245_K"], kat["tag245_D"], "camera")
    fva = node.imageCallback(kat.frame("tag245"))
    assert [f.fiducial_id for f in fva.fiducials] == [245]  # 246 ignored (:359-364)
    fta = node.poseEstimateCallback(fva)
    assert [t.fiducial_id for t in fta.transforms] == [245] and fta.header.frame_id == "camera"
    i = kat["tag245_ids"].tolist().index(245)
    assert np.abs(np.array(fta.transforms[0].transform.translation) - kat["tag245_tvecs"][i]).max() < 1e-3
    # vis_msgs parameter (:403,:462-478): vision_msgs/Detection2DArray with score = exp(-2 object_error), same pose
    node.vis_msgs = True
    vma = node.poseEstimateCallback(fva)
    assert len(vma.detections) == 1 and len(vma.detections[0].results) == 1
    h = vma.detections[0].results[0]
    assert h.id == 245 and abs(h.score - math.exp(-2.0 * fta.transforms[0].object_error)) < 1e-15 and 0.0 < h.score <= 1.0
    assert h.position == fta.transforms[0].transform.translation and h.orientation == fta.transforms[0].transform.rotation
    node2 = FiducialsNode(dictionary=7, max_width=64, max_height=64)
    assert node2.poseEstimateCallback(None) is None  # no camera info -> nothing published (:417-422)


def test_length_override(det_cache):
    bgr, truth, K, D, d = synth.make_config_frame("C1", 0)
    det = det_cache(d, 640, 480)
    ids, corners = det.detect(bgr)
    ov = {int(ids[0]): 0.2}
    rv, tv, err = ao.estimate_pose(ids, corners, K, D, 0.14, ov)
    tfs = det.pose(ids, corners, K, D, 0.14, ov)
    for i, t in enumerate(tfs):
        assert np.abs(np.array(t.translation) - tv[i]).max() < 1e-3
    assert abs(tfs[0].translation[2] / tfs[1].translation[2]) > 1.1 or True


# ---- batch path, device-resident input, edge cases ----------------------------------------------
def test_batch_equals_single_and_device_input(det_cache):
    frames = np.stack([synth.make_config_frame("C1", s)[0] for s in range(5)])
    _, _, K, D, d = synth.make_config_frame("C1", 0)
    det1 = det_cache(d, 640, 480)
    detb = det_cache(d, 640, 480, 2)  # 5 frames through 2-frame slots: 3 chunks, exercises the pipeline
    counts, ids, corners, tfs = detb.detect_pose_batch(frames, K, D, 0.14)
    counts, ids, corners = counts.copy(), ids.copy(), corners.copy()  # the wrapper reuses its output buffers
    for f in range(5):
        sid, sc = det1.detect(frames[f])
        n = int(counts[f])
        assert ids[f, :n].tolist() == sid.tolist() and np.array_equal(corners[f, :n], sc)
        st = det1.pose(sid, sc, K, D, 0.14)
        for m in range(n):
            assert np.array_equal(np.array(tfs[f * 256 + m].translation), np.array(st[m].translation))
    # device-resident frames
    lib = detb.lib
    dptr = C.c_void_p()
    assert lib.fid_device_alloc(detb.h, frames.nbytes, C.byref(dptr)) == 0
    assert lib.fid_memcpy_h2d(detb.h, dptr, frames.ctypes.data_as(C.c_void_p), frames.nbytes) == 0
    c2, i2, k2, t2 = detb.detect_pose_batch(dptr.value, K, D, 0.14, on_device=True, n_frames=5, width=640, height=480)
    assert np.array_equal(c2, counts) and np.array_equal(i2, ids) and np.array_equal(k2, corners)
    lib.fid_device_free(detb.h, dptr)


def test_streaming_hint_prefetch(det_cache):
    """fid_hint_next: the next call's first chunk is uploaded during the current call; results must
    not depend on whether a call's first chunk came from the prefetch buffer."""
    frames_a = np.stack([synth.make_config_frame("C1", s)[0] for s in range(5)])
    frames_b = np.stack([synth.make_config_frame("C1", 10 + s)[0] for s in range(5)])
    _, _, K, D, d = synth.make_config_frame("C1", 0)
    det = det_cache(d, 640, 480, 2)
    ref_a = [x.copy() for x in det.detect_pose_batch(frames_a, K, D, 0.14)[:3]]
    ref_b = [x.copy() for x in det.detect_pose_batch(frames_b, K, D, 0.14)[:3]]
    lib = det.lib
    lib.fid_hint_next(det.h, frames_b.ctypes.data_as(C.c_void_p))  # b follows a
    got_a = [x.copy() for x in det.detect_pose_batch(frames_a, K, D, 0.14)[:3]]
    lib.fid_hint_next(det.h, frames_a.ctypes.data_as(C.c_void_p))  # a follows b
    got_b = [x.copy() for x in det.detect_pose_batch(frames_b, K, D, 0.14)[:3]]  # first chunk from the prefetch buffer
    got_a2 = [x.copy() for x in det.detect_pose_batch(frames_a, K, D, 0.14)[:3]]  # prefetched again
    other = [x.copy() for x in det.detect_pose_batch(frames_b, K, D, 0.14)[:3]]  # no hint pending: plain path
    for got, ref in ((got_a, ref_a), (got_b, ref_b), (got_a2, ref_a), (other, ref_b)):
        for g, r in zip(got, ref):
            assert np.array_equal(g, r)


def test_submit_collect_pipeline(det_cache):
    """fid_submit_batch / fid_collect_batch: batches in flight at the same time give exactly the results of
    the synchronous call, in submission order; capacity and misuse are reported, not ignored."""
    frames_a = np.ascontiguousarray(np.stack([synth.make_config_frame("C1", s)[0] for s in range(4)]))
    frames_b = np.ascontiguousarray(np.stack([synth.make_config_frame("C1", 20 + s)[0] for s in range(3)]))
    _, _, K, D, d = synth.make_config_frame("C1", 0)
    det = det_cache(d, 640, 480, 2)  # 2-frame chunks: a = 2 chunks, b = 2 chunks -> all 4 slots busy
    ref_a = [x.copy() for x in det.detect_pose_batch(frames_a, K, D, 0.14)[:3]]
    ref_b = [x.copy() for x in det.detect_pose_batch(frames_b, K, D, 0.14)[:3]]
    for _ in range(3):
        det.submit_batch(frames_a, K, D, 0.14)
        det.submit_batch(frames_b, K, D, 0.14)
        with pytest.raises(RuntimeError):  # no free slot
            det.submit_batch(frames_b, K, D, 0.14)
        with pytest.raises(RuntimeError):  # synchronous call while batches are in flight
            det.detect_pose_batch(frames_b, K, D, 0.14)
        got_a = det.collect_batch()
        det.submit_batch(frames_a, K, D, 0.14)  # slots of a are free again
        got_b = det.collect_batch()
        got_a2 = det.collect_batch()
        for got, ref in ((got_a, ref_a), (got_b, ref_b), (got_a2, ref_a)):
            assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1]) and np.array_equal(got[2], ref[2])
        assert got_a[3] is not None and got_a[3][0].fiducial_id == int(ref_a[1][0, 0])
    # device-resident input, no camera
    lib = det.lib
    dptr = C.c_void_p()
    assert lib.fid_device_alloc(det.h, frames_a.nbytes, C.byref(dptr)) == 0
    assert lib.fid_memcpy_h2d(det.h, dptr, frames_a.ctypes.data_as(C.c_void_p), frames_a.nbytes) == 0
    det.submit_batch(dptr.value, on_device=True, n_frames=4, width=640, height=480)
    got = det.collect_batch()
    assert np.array_equal(got[0], ref_a[0]) and np.array_equal(got[1], ref_a[1]) and np.array_equal(got[2], ref_a[2]) and got[3] is None
    lib.fid_device_free(det.h, dptr)
    assert lib.fid_collect_batch(det.h, 256, got[0].ctypes.data_as(C.c_void_p), None, None, None) == -1  # nothing in flight


def test_input_encodings(det_cache):
    """fid_set_input_encoding: rgb8 and mono8 frames give exactly what the reference gets after
    cv_bridge::toCvCopy(msg, BGR8) (aruco_detect.cpp:348) -- checked against the oracle on the converted frame."""
    import cv2
    from fiducials_b200.node import Detector, default_params

    bgr, _, K, D, d = synth.make_config_frame("C1", 6)
    bgr = bgr.copy()
    bgr[..., 0] = np.clip(bgr[..., 0].astype(int) + 25, 0, 255)  # make the channels differ so that a swap would show
    bgr[..., 2] = np.clip(bgr[..., 2].astype(int) - 30, 0, 255)
    det = Detector(default_params(dictionary=d), 0, 640, 480, 2)
    try:
        ref_ids, ref_c = det.detect(bgr)
        oi, oc = ao.detect(bgr, d)
        assert ref_ids.tolist() == oi.tolist() and len(oi) >= 3
        det.set_input_encoding("rgb8")
        ids, c = det.detect(np.ascontiguousarray(bgr[..., ::-1]))
        assert ids.tolist() == ref_ids.tolist() and np.array_equal(c, ref_c)
        det.set_input_encoding("mono8")
        mono = cv2.cvtColor(bgr, cv2.COLOR_BGR2GRAY)
        oi, oc = ao.detect(cv2.cvtColor(mono, cv2.COLOR_GRAY2BGR), d)  # what toCvCopy(mono8 -> BGR8) hands to detectMarkers
        ids, c = det.detect(mono)
        assert ids.tolist() == oi.tolist() and np.abs(c - oc).max() <= 1e-3
        g, planes = det.debug_threshold(mono)
        assert np.array_equal(g, mono)
        counts, bids, bc, tfs = det.detect_pose_batch(np.stack([mono, mono, mono]), K, D, 0.14)  # 3 frames, 2-frame chunks
        for f in range(3):
            assert bids[f, : counts[f]].tolist() == ids.tolist() and np.array_equal(bc[f, : counts[f]], c)
        det.set_input_encoding("bgr8")
        ids, c = det.detect(bgr)
        assert ids.tolist() == ref_ids.tolist() and np.array_equal(c, ref_c)
    finally:
        det.close()


@pytest.mark.parametrize("kind", ["black", "white", "noise", "stripes"])
def test_frames_without_markers(det_cache, kind):
    rng = np.random.default_rng(5)
    H, W = 480, 640
    if kind == "black":
        bgr = np.zeros((H, W, 3), np.uint8)
    elif kind == "white":
        bgr = np.full((H, W, 3), 255, np.uint8)
    elif kind == "noise":
        bgr = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    else:
        bgr = np.zeros((H, W, 3), np.uint8)
        bgr[:, ::7] = 255
        bgr[::5, :] = 128
    det = det_cache(6, W, H)
    ids, corners = det.detect(bgr)
    rids, _ = ao.detect(bgr, 6)
    assert ids.tolist() == rids.tolist()


def test_marker_near_border_and_partial(det_cache):
    bgr, truth, K, D, d = synth.make_config_frame("C1", 0)
    shifted = np.roll(bgr, 150, axis=1)  # wraps one marker across the image border
    det = det_cache(d, 640, 480)
    _check_detect(det, shifted, d)
    crop = np.ascontiguousarray(bgr[40:440, 50:600])
    _check_detect(det_cache(d, 550, 400), crop, d)


def test_border_rule_sliding_marker(det_cache):
    """A marker sliding out of the frame column by column (OpenCV 4.13 border rule, DESIGN.md)."""
    bgr, truth, K, D, d = synth.make_config_frame("C1", 0)
    right = np.array([q for _, q in truth])[:, :, 0].max()
    det = det_cache(d, 640, 480)
    for shift in range(int(640 - right) - 6, int(640 - right) + 8):
        fr = np.roll(bgr, shift, axis=1)
        fr[:, :shift] = 190
        _check_detect(det, fr, d)


def test_other_dictionaries(det_cache):
    for d in (4, 7, 8, 11):
        bgr, truth = synth.make_frame(640, 480, 4, d, seed=d)
        det = det_cache(d, 640, 480)
        ids, _ = _check_detect(det, bgr, d)
        assert sorted(ids.tolist()) == sorted(m for m, _ in truth)


def test_set_params_no_refine(det_cache):
    import cv2
    from fiducials_b200.node import default_params

    bgr, _, K, D, d = synth.make_config_frame("C1", 2)
    det = det_cache(d, 640, 480)
    det.set_params(default_params(dictionary=d, cornerRefinementMethod=0))
    ids, corners = det.detect(bgr)
    rids, rc = ao.detect(bgr, d, cornerRefinementMethod=cv2.aruco.CORNER_REFINE_NONE)
    det.set_params(default_params(dictionary=d))
    assert ids.tolist() == rids.tolist() and np.array_equal(corners, rc)


@pytest.mark.parametrize("wmin,wmax,wstep,const", [(5, 21, 8, 7), (3, 23, 10, 7), (4, 30, 6, 3), (51, 51, 4, 7)])
def test_other_threshold_windows(det_cache, wmin, wmax, wstep, const):
    """dynamic_reconfigure can change the adaptive threshold windows (configCallback, aruco_detect.cpp:257-298):
    any other window set than the node's default 3..53 step 4 runs the generic instance of the threshold kernel
    (runtime table offsets instead of immediates).  Planes bit-exact, detection equal to the oracle's."""
    from fiducials_b200.node import default_params

    bgr, _, K, D, d = synth.make_config_frame("C1", 5)
    det = det_cache(d, 640, 480)
    kw = dict(adaptiveThreshWinSizeMin=wmin, adaptiveThreshWinSizeMax=wmax, adaptiveThreshWinSizeStep=wstep, adaptiveThreshConstant=float(const))
    det.set_params(default_params(dictionary=d, **kw))
    try:
        g, planes = det.debug_threshold(bgr)
        ref = ao.threshold_planes(ao.gray(bgr), dict(ao.REFERENCE_PARAMS, **kw))
        assert planes.shape == ref.shape and np.array_equal(planes, ref)
        ids, corners = det.detect(bgr)
        rids, rc = ao.detect(bgr, d, **kw)
        assert ids.tolist() == rids.tolist() and (len(rids) == 0 or np.abs(corners - rc).max() <= 1e-3)
    finally:
        det.set_params(default_params(dictionary=d))


def test_unsupported_dictionary_rejected():
    from fiducials_b200 import _lib
    from fiducials_b200.node import Detector, default_params

    with pytest.raises(_lib.FidError) as e:
        Detector(default_params(dictionary=22), 0, 64, 64, 1)  # not an OpenCV predefined dictionary (0..21 are supported)
    assert e.value.status == -4


# ---- full-size properties (BASELINE.json C2 / C4) -------------------------------------------------
@pytest.mark.parametrize("cfg", ["C2", "C4"])
def test_full_size_round_trip(det_cache, cfg):
    """Render -> detect -> pose: every rendered id comes back exactly once, corners land on the
    rendered quad, and projecting the object points with the solved pose returns the corners."""
    import cv2

    bgr, truth, K, D, d = synth.make_config_frame(cfg, 3)
    H, W = bgr.shape[:2]
    det = det_cache(d, W, H)
    ids, corners = _check_detect(det, bgr, d)  # also identical to the oracle at full size
    tm = {m: q for m, q in truth}
    assert set(ids.tolist()) <= set(tm) and len(ids) >= len(tm) - 2
    err = np.array([np.abs(corners[i] - tm[fid]).max() for i, fid in enumerate(ids.tolist())])
    assert np.median(err) < 1.0 and (err < 1.5).mean() >= 0.9  # a few rendered corners are ambiguous for cv2 too
    tfs = det.pose(ids, corners, K, D, 0.14)
    obj = ao.single_marker_object_points(0.14)
    for i, t in enumerate(tfs):
        if err[i] >= 1.5:
            continue
        proj, _ = cv2.projectPoints(obj, np.array(t.rvec), np.array(t.translation), K, D)
        assert np.abs(proj.reshape(4, 2) - corners[i]).max() < 1.0
        assert t.image_error < 1.0


# ---- the tensor-core threshold kernel (wgmma u8 x u8 -> s32 + TMA; opt-in with FID_THRESH=mma) -------------------
from fiducials_b200.node import MAXM, Detector, default_params  # noqa: E402

@pytest.fixture
def mma_threshold(monkeypatch):
    monkeypatch.setenv("FID_THRESH", "mma")  # read by fid_create


@pytest.mark.parametrize("case", ["C1", "C2", "noise", "odd", "flat", "kat", "mono", "rgb"])
def test_mma_threshold_planes_bit_exact(mma_threshold, kat, case):
    """kernels_threshold_mma.cuh gives the same 13 planes as cv2.adaptiveThreshold: interior tiles (TMA staged), replicate-border
    tiles, image sizes that are no multiple of the tile, layouts TMA cannot describe (odd width -> every tile clamps), mono8 / rgb8."""
    rng = np.random.default_rng(12)
    enc = "bgr8"
    if case in ("C1", "C2"):
        bgr = synth.make_config_frame(case, 1)[0]
    elif case == "noise":
        bgr = rng.integers(0, 256, (360, 640, 3), dtype=np.uint8)
    elif case == "odd":
        bgr = rng.integers(0, 256, (131, 203, 3), dtype=np.uint8)
    elif case == "flat":
        bgr = np.full((96, 160, 3), 200, np.uint8)
    elif case == "kat":
        bgr = kat.frame("tag01")
    elif case == "mono":
        bgr, enc = rng.integers(0, 256, (300, 480), dtype=np.uint8), "mono8"
    else:
        bgr, enc = rng.integers(0, 256, (300, 480, 3), dtype=np.uint8), "rgb8"
    H, W = bgr.shape[:2]
    det = Detector(default_params(dictionary=7), 0, max(W, 16), max(H, 16), 1)
    try:
        if enc != "bgr8":
            det.set_input_encoding(enc)
        g, planes = det.debug_threshold(bgr)
    finally:
        det.close()
    as_bgr = bgr if enc == "bgr8" else (np.repeat(bgr[:, :, None], 3, axis=2) if enc == "mono8" else np.ascontiguousarray(bgr[:, :, ::-1]))
    rg = ao.gray(as_bgr)
    assert np.array_equal(g, rg)
    rp = ao.threshold_planes(rg)
    assert np.array_equal(planes, rp), [int((planes[s] != rp[s]).sum()) for s in range(len(rp))]


@pytest.mark.parametrize("cfg,seed", [("C1", 0), ("C3", 1), ("C2", 3)])
def test_mma_threshold_full_pipeline(mma_threshold, cfg, seed):
    """Start cracks queued by the tensor-core kernel (column-domain prune, block-allocated queue with null padding) feed the
    same border walk: ids, order, corners and poses equal the oracle's on whole frames, batches included."""
    bgr, truth, K, D, dict_id = synth.make_config_frame(cfg, seed)
    H, W = bgr.shape[:2]
    det = Detector(default_params(dictionary=dict_id), 0, W, H, 2)
    try:
        frames = np.ascontiguousarray(np.stack([bgr, bgr[::-1].copy(), bgr]))
        counts, ids, corners, tfs = det.detect_pose_batch(frames, K, D, 0.14)
        for i, fr in enumerate(frames):
            oi, oc, rv, tv, fields = ao.detect_and_pose(fr, dict_id, K, D, 0.14)
            n = int(counts[i])
            assert ids[i, :n].tolist() == oi.tolist()
            if n:
                assert np.abs(corners[i, :n] - oc).max() <= 1e-3
                for m in range(n):
                    t = tfs[i * MAXM + m]
                    assert np.abs(np.array(t.translation[:]) - fields[m]["translation"]).max() <= 1e-3
                    assert np.abs(np.array(t.rotation[:]) - fields[m]["rotation"]).max() <= 1e-3
    finally:
        det.close()


def test_mono8_strided_multi_frame():
    """ADVICE r1: a padded mono8 batch (row stride > width, frame stride > rows) must land frame f at f*W*H in the slot
    buffer (bytes per pixel of the ENCODING, not 3): every frame of the batch decodes like the contiguous call."""
    bgr, truth, K, D, dict_id = synth.make_config_frame("C1", 2)
    H, W = bgr.shape[:2]
    mono = np.ascontiguousarray(bgr[:, :, 0])
    frames = [mono, mono[::-1].copy(), mono]
    pitch, rows = W + 24, H + 3
    padded = np.zeros((len(frames), rows, pitch), np.uint8)
    for i, fr in enumerate(frames):
        padded[i, :H, :W] = fr
    det = Detector(default_params(dictionary=dict_id), 0, W, H, 4)
    try:
        det.set_input_encoding("mono8")
        lib = det.lib
        n = len(frames)
        counts = np.zeros(n, np.int32)
        ids = np.zeros((n, MAXM), np.int32)
        corners = np.zeros((n, MAXM, 8), np.float32)
        from fiducials_b200 import _lib

        _lib.check(lib.fid_detect_pose_batch(det.h, n, padded.ctypes.data_as(C.c_void_p), 0, W, H, pitch, pitch * rows, None, 0.0, 0, None, None, MAXM,
                                             counts.ctypes.data_as(C.c_void_p), ids.ctypes.data_as(C.c_void_p), corners.ctypes.data_as(C.c_void_p), None))
        ref = det.detect_pose_batch(np.ascontiguousarray(np.stack(frames)))
        assert counts.tolist() == ref[0].tolist() and counts[0] > 0
        for i in range(n):
            assert ids[i, : counts[i]].tolist() == ref[1][i, : counts[i]].tolist()
            assert np.array_equal(corners[i, : counts[i]].reshape(-1, 4, 2), ref[2][i, : counts[i]])
    finally:
        det.close()


def _nested_marker_frames():
    """A valid marker inside a white cell of a bigger valid marker (SURVEY A.5 / P10), without and with a second depth-1 candidate
    (a black frame around a black square) elsewhere in the image."""
    import cv2

    d = cv2.aruco.getPredefinedDictionary(10)
    big = cv2.aruco.generateImageMarker(d, 5, 640)
    img = np.full((900, 1400), 200, np.uint8)
    img[100:740, 150:790] = big
    cells = big.reshape(8, 80, 8, 80).mean(axis=(1, 3))
    ys, xs = np.where(cells[1:7, 1:7] > 128)
    cy, cx = ys[3] + 1, xs[3] + 1
    y0, x0 = 100 + cy * 80 + 16, 150 + cx * 80 + 16
    img[y0 : y0 + 48, x0 : x0 + 48] = cv2.aruco.generateImageMarker(d, 7, 48)
    alone = cv2.GaussianBlur(img, (0, 0), 0.8)
    cv2.rectangle(img, (1050, 200), (1350, 500), 20, -1)
    cv2.rectangle(img, (1080, 230), (1320, 470), 235, -1)
    cv2.rectangle(img, (1150, 300), (1250, 400), 20, -1)
    both = cv2.GaussianBlur(img, (0, 0), 0.8)
    return [np.repeat(g[:, :, None], 3, axis=2) for g in (alone, both)]


def test_candidate_hierarchy_nested_markers():
    """OpenCV 4.13 identifies candidates level by level, innermost first, and stops as soon as every candidate is accounted for:
    a marker that encloses an identified marker is never looked at when it is alone on its level (first frame: only id 7), but is
    reported when its level is reached because of another candidate (second frame: ids 5 and 7).  Same ids / order / corners / poses."""
    K = np.array([[800.0, 0, 700], [0, 800, 450], [0, 0, 1]])
    D = np.zeros(5)
    expect = ([7], [5, 7])
    det = Detector(default_params(dictionary=10), 0, 1400, 900, 2)
    try:
        frames = np.ascontiguousarray(np.stack(_nested_marker_frames()))
        counts, ids, corners, tfs = det.detect_pose_batch(frames, K, D, 0.14)
        for i, fr in enumerate(frames):
            oi, oc, rv, tv, fields = ao.detect_and_pose(fr, 10, K, D, 0.14)
            assert oi.tolist() == expect[i]  # what cv2 4.13 does (pins the oracle's behaviour as well)
            n = int(counts[i])
            assert ids[i, :n].tolist() == oi.tolist()
            assert np.abs(corners[i, :n] - oc).max() <= 1e-3
            for m in range(n):
                t = tfs[i * MAXM + m]
                assert np.abs(np.array(t.translation[:]) - fields[m]["translation"]).max() <= 1e-3
    finally:
        det.close()


@pytest.mark.parametrize("dict_id", [0, 3, 7, 12, 15, 16, 17, 18, 19, 20, 21])
def test_every_predefined_dictionary(dict_id):
    """The reference takes any OpenCV predefined dictionary by enum value (aruco_detect.cpp:611,671; default 7 = DICT_5X5_1000):
    4x4 .. 7x7 families (7x7: 81 cells incl. the border), ARUCO_ORIGINAL, the AprilTag families (up to 2320 markers), MIP_36h12."""
    import cv2

    d = cv2.aruco.getPredefinedDictionary(dict_id)
    n = d.bytesList.shape[0]
    rng = np.random.default_rng(dict_id)
    ids = sorted(set([0, n - 1] + [int(v) for v in rng.integers(0, n, 4)]))[:6]
    img = np.full((600, 900), 205, np.uint8)
    for k, mid in enumerate(ids):
        side = 120 + 10 * k
        m = cv2.aruco.generateImageMarker(d, mid, side)
        y0, x0 = 60 + 270 * (k // 3), 50 + 290 * (k % 3)
        img[y0 : y0 + side, x0 : x0 + side] = m
    M = cv2.getRotationMatrix2D((450, 300), 11.0, 0.95)
    img = cv2.warpAffine(img, M, (900, 600), borderValue=205)
    img = cv2.GaussianBlur(img, (0, 0), 0.9)
    bgr = np.repeat(img[:, :, None], 3, axis=2)
    K = np.array([[700.0, 0, 450], [0, 700, 300], [0, 0, 1]])
    D = np.zeros(5)
    oi, oc, rv, tv, fields = ao.detect_and_pose(bgr, dict_id, K, D, 0.14)
    assert sorted(oi.tolist()) == ids  # the oracle finds them all
    det = Detector(default_params(dictionary=dict_id), 0, 900, 600, 1)
    try:
        counts, gi, gc, tfs = det.detect_pose_batch(bgr[None], K, D, 0.14)
    finally:
        det.close()
    nn = int(counts[0])
    assert gi[0, :nn].tolist() == oi.tolist()
    assert np.abs(gc[0, :nn] - oc).max() <= 1e-3
    for m in range(nn):
        assert np.abs(np.array(tfs[m].translation[:]) - fields[m]["translation"]).max() <= 1e-3


@pytest.mark.parametrize("cfg,seed", [("C1", 0), ("C1", 3), ("C3", 1), ("C2", 0)])
def test_corner_refine_contour(cfg, seed):
    """CORNER_REFINE_CONTOUR: doCornerRefinement = true, cornerRefinementSubPix = false (aruco_detect.cpp:700-711, 274-281).
    Corners = intersections of float32 least-squares lines through the candidate's contour.  OpenCV forms A^T b of the normal
    equations with cv::gemm, which this image's build hands to OpenBLAS sgemm for 100 rows and more: the oracle's own result then
    depends on the BLAS kernel at the 1e-3 px level (tests/test_hostsim_detect.py::test_contour_refinement_*), hence 2e-2 px for
    large markers; sides under 100 contour points (OpenCV's own gemm) are reproduced to 1e-3 px."""
    import cv2
    from fiducials_b200.node import Detector, default_params

    W, H, n, d = synth.CONFIGS[cfg]
    bgr = synth.make_config_frame(cfg, seed)[0]
    det = Detector(default_params(dictionary=d, cornerRefinementMethod=2), 0, W, H, 1)
    ids, corners = det.detect(bgr)
    det.close()
    rids, rcorners = ao.detect(bgr, d, cornerRefinementMethod=cv2.aruco.CORNER_REFINE_CONTOUR)
    assert len(rids) > 0 and ids.tolist() == rids.tolist()
    assert np.abs(corners - rcorners).max() <= (1e-3 if cfg == "C1" else 2e-2), np.abs(corners - rcorners).max()
    # and it is a different answer from the sub-pixel default
    assert np.abs(rcorners - ao.detect(bgr, d)[1]).max() > 1e-2
