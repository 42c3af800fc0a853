"""The contour stage (start-crack queue, k_walk rounds, k_emit, k_approx*) on the frames of tests/contour_cases.py against cv2: fine
textures that fill the start-crack queue past its size, contours decided only in the persistent walk round, markers and blobs on the
halo-tile seams and the frame borders, contours at the length filter's bounds, and frames past the chain and point capacities.
The start-crack and in-range contour counters equal the CPU's counts.
Every case runs with the default threshold kernel, the tensor-core one (FID_THRESH=mma) and the table pruning of the start cracks
(FID_START_PRUNE=1).  Tolerances as in tests/test_gpu_parity.py: candidates bit-exact, ids and order identical, corners within 1e-3 px."""
import ctypes as C
import functools

import numpy as np
import pytest

import contour_cases as cc
import hostsim_util as hs
from fiducials_b200 import synth
from fiducials_b200.node import MAXM, Detector, FiducialsNode, default_params
from oracle import aruco_oracle as ao

pytestmark = pytest.mark.gpu

FID_OK, FID_ERR_CAPACITY = 0, -5
FID_MAX_RAW = 4096
# the texture cases run here; the full-frame 1-pixel patterns at 1080p and above cost cv2 minutes per frame and add nothing the
# 640 x 480 ones and the half-frame ones do not cover
TEXTURE_CASES = [f"{t}_{l}_vga" for t in cc.TEXTURES for l in ("full", "half")] + [
    "checker1_half_fhd", "dither1_half_fhd", "checker2_full_fhd", "noise_full_fhd", "checker1_half_uhd"]
SHAPE_CASES = ["spiral_fhd", "serpentine_fhd", "seams_599x449", "seams_600x450", "seams_601x451", "seams_1919x1079", "seams_1921x1081",
               "borders_fhd", "length_min_vga", "length_max_vga"]
CAPACITY_CASES = ["segments_hd_in_uhd", "lines_fhd"]  # past max_chains, past max_points: FID_ERR_CAPACITY


@pytest.fixture(params=["simt", "mma", "prune"])
def mode(request, monkeypatch):
    """The threshold kernels and the start pruning (read by fid_create)."""
    monkeypatch.delenv("FID_THRESH", raising=False)
    monkeypatch.delenv("FID_START_PRUNE", raising=False)
    if request.param == "mma":
        monkeypatch.setenv("FID_THRESH", "mma")
    elif request.param == "prune":
        monkeypatch.setenv("FID_START_PRUNE", "1")
    return request.param


@functools.lru_cache(maxsize=None)
def _oracle(name):
    """cv2's ids and corners of a case."""
    return ao.detect(cc.render(name)[0], cc.DICT)


@functools.lru_cache(maxsize=None)
def _cpu_counts(name):
    """(start cracks, in-range contours) of a case, counted on the CPU: the start rules restated in numpy, and the host build of the
    walk, which lists cv2.findContours' contours (tests/test_hostsim_contours.py), between the detector's min_len and max_len."""
    c = cc.CASES[name]
    planes = ao.threshold_planes(ao.gray(cc.render(name)[0]))
    lo, hi = cc.min_len(c["W"], c["H"]), cc.max_len(c["W"], c["H"])
    return int(cc.start_counts(planes).sum()), sum(len(hs.find_contours(p, lo, hi)[0]) for p in planes)


@functools.lru_cache(maxsize=None)
def _raw(name):
    """cv2's raw quad candidates of a case (oracle.aruco_oracle.quad_candidates)."""
    return ao.quad_candidates(ao.gray(cc.render(name)[0]))


def _raw_detect(det, bgr):
    """fid_detect through ctypes (the wrapper raises on a nonzero status): (status, ids, corners [n, 4, 2])."""
    H, W = bgr.shape[:2]
    ids = np.full(MAXM, -7, np.int32)
    corners = np.zeros((MAXM, 8), np.float32)
    n = C.c_int(-1)
    st = det.lib.fid_detect(det.h, bgr.ctypes.data_as(C.c_void_p), W, H, W * 3, MAXM, C.byref(n), ids.ctypes.data_as(C.c_void_p),
                            corners.ctypes.data_as(C.c_void_p))
    return st, ids[: max(n.value, 0)].copy(), corners[: max(n.value, 0)].reshape(-1, 4, 2).copy()


def _detector(W, H, max_batch=1):
    return Detector(default_params(dictionary=cc.DICT), 0, W, H, max_batch)


def _assert_cv2(ids, corners, name):
    rids, rcorners = _oracle(name)
    assert ids.tolist() == rids.tolist(), (name, ids.tolist(), rids.tolist())
    if len(rids):
        assert np.abs(corners - rcorners).max() <= 1e-3, name


@pytest.mark.parametrize("name", TEXTURE_CASES + SHAPE_CASES)
def test_contour_stage_matches_cv2(mode, name):
    """The frame's markers are cv2's; its raw candidates are cv2's bit for bit; the in-range contour counter is the CPU's, and so is
    the start-crack counter with the default kernel (the tensor-core kernel pads its queue blocks, the pruning drops starts)."""
    bgr, rendered = cc.render(name)
    c = cc.CASES[name]
    det = _detector(c["W"], c["H"])
    try:
        st, ids, corners = _raw_detect(det, bgr)
        assert st == FID_OK, (name, st)
        _assert_cv2(ids, corners, name)
        assert set(ids.tolist()) == rendered or c["kind"] == "borders", name
        starts, chains = _cpu_counts(name)
        cnt = det.last_counters()
        assert cnt["contours_in_range"] == chains, (name, cnt, chains)
        if mode == "simt":
            assert cnt["start_cracks"] == starts, (name, cnt, starts)
        if c["kind"] == "texture" and c["W"] > 640:
            return  # cv2's candidate stage on these frames costs minutes (millions of contours); the 640 x 480 ones cover it
        raw = _raw(name)
        if len(raw) <= FID_MAX_RAW:
            quads, scale, clen = det.debug_candidates()
            assert len(quads) == len(raw), (name, len(quads), len(raw))
            assert np.array_equal(scale, [s for s, _, _ in raw]) and np.array_equal(clen, [n for _, _, n in raw]), name
            assert np.array_equal(quads, np.array([q for _, q, _ in raw]).reshape(-1, 4, 2)), name
    finally:
        det.close()


@pytest.mark.parametrize("name", CAPACITY_CASES)
def test_capacity_reported_and_markers_are_cv2s(mode, name):
    """Past the chain capacity (65 536 in-range contours per frame) or the point capacity (4 W H + 65 536 in-range contour points of
    the handle's frame size): the status says so, and every marker returned is one cv2 returns, with cv2's corners."""
    bgr, _ = cc.render(name)
    rids, rcorners = _oracle(name)
    det = _detector(*cc.handle(name))
    try:
        st, ids, corners = _raw_detect(det, bgr)
    finally:
        det.close()
    assert st == FID_ERR_CAPACITY, (name, st)
    ref = {int(i): k for k, i in enumerate(rids)}
    assert len(set(ids.tolist())) == len(ids) and set(ids.tolist()) <= set(ref), name
    for i, q in zip(ids.tolist(), corners):
        assert np.abs(q - rcorners[ref[i]]).max() <= 1e-3, (name, i)


def _single(det, bgr):
    counts, ids, corners, _ = det.detect_pose_batch(bgr[None])
    n = int(counts[0])
    return ids[0, :n].copy(), corners[0, :n].copy()


@pytest.mark.parametrize("max_batch", [2, 4])
def test_batch_frames_independent_of_their_neighbours(mode, max_batch):
    """Overflowing frames in chunks of 2 and 4 next to C2 frames (and next to each other): each frame's result is its single-frame
    result and cv2's, and the call succeeds whatever the chunk holds."""
    c2 = [synth.make_config_frame("C2", s)[0] for s in (3, 4)]
    tex = [cc.render(n)[0] for n in ("checker1_half_fhd", "dither1_half_fhd")]
    frames = np.ascontiguousarray(np.stack([tex[0], c2[0], tex[1], tex[0], c2[1], c2[0], tex[1], tex[0]]))
    one = _detector(1920, 1080)
    det = _detector(1920, 1080, max_batch)
    try:
        singles = [_single(one, f) for f in frames]
        counts, ids, corners, _ = det.detect_pose_batch(frames)
    finally:
        one.close()
        det.close()
    for f in range(len(frames)):
        n = int(counts[f])
        assert ids[f, :n].tolist() == singles[f][0].tolist(), f
        assert np.array_equal(corners[f, :n], singles[f][1]), f
    for f, name in ((0, "checker1_half_fhd"), (2, "dither1_half_fhd")):
        _assert_cv2(ids[f, : counts[f]], corners[f, : counts[f]], name)


def test_node_publishes_markers_of_an_overflowing_frame(mode):
    """FiducialsNode.imageCallback on the half-checkerboard frame: the frame is not dropped, and it publishes cv2's markers."""
    bgr, _ = cc.render("checker1_half_fhd")
    rids, rcorners = _oracle("checker1_half_fhd")
    node = FiducialsNode(dictionary=cc.DICT, fiducial_len=0.14, max_width=1920, max_height=1080)
    fva = node.imageCallback(bgr)
    assert fva is not None
    assert [f.fiducial_id for f in fva.fiducials] == rids.tolist()
