"""useAruco3Detection on the device (fid_set_aruco3, fid_debug_aruco3_planes, fid_detect and the batch calls): the planes bit for bit
against cv2.resize / cv2.pyrDown, markers bit for bit against the host chain (tests/hostsim/aruco3_hostsim.cpp) and ids against cv2's
detectMarkers with the mode on; poses and pose hypotheses against the stand-alone calls; the mode switched off again; the refusals."""
import ctypes as C

import numpy as np
import pytest

from fiducials_b200 import _lib, synth
from fiducials_b200.board import charuco_board, grid_board
from fiducials_b200.node import MAXM, Detector, default_params
import aruco3_oracle as a3

pytestmark = pytest.mark.gpu
FID_ERR_UNSUPPORTED = -4
A = a3.A
GOLDEN = ["bag", "img403", "tag01", "tag245"]


def _det(W, H, min_side=32, ratio=0.02, dictionary=A.DICT_6X6_250, max_batch=4):
    d = Detector(default_params(dictionary=dictionary), max_width=W, max_height=H, max_batch=max_batch)
    d.set_aruco3(min_side, ratio)
    return d


def _frames(W, H, n, seed, dictionary=A.DICT_6X6_250):
    return [a3.render(W, H, dictionary, seed + i, 12, side_range=(0.2, 0.8)) for i in range(n)]


def _planes_equal(det, bgr, min_side, ratio):
    seg, levels, closest = det.debug_aruco3_planes(bgr)
    rseg, rpyr = a3.cv2_planes(a3.ao.gray(bgr), min_side, ratio)
    assert seg.shape == rseg.shape and np.array_equal(seg, rseg)
    assert len(levels) == len(rpyr) - 1
    for l, (a, b) in enumerate(zip(levels, rpyr[1:])):
        assert np.array_equal(a, b), l + 1
    assert closest == a3.geometry(bgr.shape[1], bgr.shape[0], min_side, ratio)[3]


@pytest.mark.parametrize("min_side,ratio", [(32, 0.02), (16, 0.05), (64, 0.0), (32, 0.01)])
def test_planes_match_cv2(kat, min_side, ratio):
    for name in GOLDEN:
        bgr = kat.frame(name)
        det = _det(bgr.shape[1], bgr.shape[0], min_side, ratio, max_batch=1)
        _planes_equal(det, bgr, min_side, ratio)
    for W, H in [(1921, 1079), (3840, 2160)]:
        det = _det(W, H, min_side, ratio, max_batch=1)
        _planes_equal(det, a3.blank_frame(W, H, 3, noise_only=True), min_side, ratio)


def _check_frame(ids, corners, bgr, dictionary, min_side, ratio, vs_cv2=True):
    hids, hcorners = a3.host_detect(bgr, dictionary, min_side, ratio)
    assert ids.tolist() == hids.tolist()
    assert np.array_equal(corners, hcorners), np.abs(corners - hcorners).max(initial=0)
    if vs_cv2:
        rids, rcorners = a3.cv2_detect(bgr, dictionary, min_side, ratio)
        assert ids.tolist() == rids.tolist()
        assert np.abs(corners - rcorners).max(initial=0) <= 0.05


def test_golden_frames(kat):
    for name in GOLDEN:
        bgr = kat.frame(name)
        for min_side, ratio in [(32, 0.02), (32, 0.0), (16, 0.05)]:
            det = _det(bgr.shape[1], bgr.shape[0], min_side, ratio, dictionary=A.DICT_5X5_1000, max_batch=1)
            ids, corners = det.detect(bgr)
            _check_frame(ids, corners, bgr, det.params.dictionary, min_side, ratio)


@pytest.mark.parametrize("W,H,ratio,dictionary", [(1920, 1080, 0.02, A.DICT_6X6_250), (1920, 1080, 0.05, A.DICT_APRILTAG_36h11), (3840, 2160, 0.02, A.DICT_6X6_250),
                                                  (3840, 2160, 0.05, A.DICT_APRILTAG_36h11)])
def test_detect_matches_host_and_cv2(W, H, ratio, dictionary):
    det = _det(W, H, 32, ratio, dictionary, max_batch=1)
    n = 0
    for bgr in _frames(W, H, 2, 100 + W // 100 + int(ratio * 100), dictionary):
        ids, corners = det.detect(bgr)
        _check_frame(ids, corners, bgr, dictionary, 32, ratio)
        n += len(ids)
    assert n >= 6


@pytest.mark.parametrize("W,H,ratio", [(1920, 1080, 0.02), (3840, 2160, 0.05)])
def test_mma_threshold_kernel(monkeypatch, W, H, ratio):
    """The tensor-core threshold kernel (FID_THRESH=mma) on the segmentation plane: a mono8 plane whose width (873, 549) is no
    multiple of 4, batched, so every tile takes the clamping load; markers bit-identical with the host chain, per frame and batch."""
    monkeypatch.setenv("FID_THRESH", "mma")  # read by fid_create
    det = _det(W, H, 32, ratio, A.DICT_6X6_250, max_batch=2)
    frames = np.stack(_frames(W, H, 2, 150 + int(ratio * 100)))
    counts, ids, corners, _ = det.detect_pose_batch(frames)
    counts, ids, corners = counts.copy(), ids.copy(), corners.copy()
    for f, bgr in enumerate(frames):
        n = counts[f]
        _check_frame(ids[f, :n], corners[f, :n], bgr, A.DICT_6X6_250, 32, ratio, vs_cv2=f == 0)
        fids, fcorners = det.detect(bgr)
        assert ids[f, :n].tolist() == fids.tolist() and np.array_equal(corners[f, :n], fcorners)
    assert counts.sum() >= 6


def test_batch_equals_frames_and_pose():
    W, H = 1920, 1080
    K, D = synth.camera_for(W, H)
    det = _det(W, H, 32, 0.02)
    frames = np.stack(_frames(W, H, 3, 300))
    counts, ids, corners, tfs = det.detect_pose_batch(frames, K, D, 0.14, {3: 0.2})
    counts, ids, corners = counts.copy(), ids.copy(), corners.copy()
    for f, bgr in enumerate(frames):
        n = counts[f]
        fids, fcorners = det.detect(bgr)
        assert ids[f, :n].tolist() == fids.tolist() and np.array_equal(corners[f, :n], fcorners)
        _check_frame(ids[f, :n], corners[f, :n], bgr, A.DICT_6X6_250, 32, 0.02, vs_cv2=False)
        ref = det.pose(fids, fcorners, K, D, 0.14, {3: 0.2})
        for m in range(n):
            assert bytes(tfs[f * _lib.FID_MAX_MARKERS + m]) == bytes(ref[m]), (f, m)


def test_pose_hypotheses_equal_standalone():
    W, H = 1920, 1080
    K, D = synth.camera_for(W, H)
    det = _det(W, H, 32, 0.02)
    det.set_pose_hypotheses(True)
    frames = np.stack(_frames(W, H, 2, 400))
    counts, ids, corners, _ = det.detect_pose_batch(frames, K, D, 0.14)
    counts, ids, corners = counts.copy(), ids.copy(), corners.copy()
    hyp = det.last_pose_hypotheses()
    for f in range(len(frames)):
        n = counts[f]
        ref = det.pose_hypotheses(ids[f, :n], corners[f, :n], K, D, 0.14)
        for m in range(n):
            assert bytes(hyp[f * _lib.FID_MAX_MARKERS + m]) == bytes(ref[m]), (f, m)


def test_boards_charuco_diamonds_equal_standalone():
    """The board, ChArUco and diamond stages of a batch read the full-resolution corners k_a3_corners wrote and the full-size frame:
    their records equal fid_estimate_board_poses / fid_detect_charuco / fid_detect_diamonds on the batch's own markers."""
    import cv2
    from test_hostsim_diamond import D_ZERO, K_SYN, RATIOS, H as DH, W as DW, scene
    import diamond_oracle as do

    rng = np.random.default_rng(21)
    sq, mk = RATIOS[0]
    frames = np.ascontiguousarray(np.stack([cv2.cvtColor(scene(rng, 2, "near", RATIOS[0])[0], cv2.COLOR_GRAY2BGR) for f in range(4)]))
    det = _det(DW, DH, 32, 0.02, do.DICT_ID)  # 800 x 600: a 533 x 400 plane, one cornerSubPix level
    det.set_boards([grid_board((2, 2), 0.03, 0.008, [240, 241, 242, 243])])
    det.set_charuco_boards([charuco_board((5, 4), 0.03, 0.022)])
    det.set_diamonds(sq, mk)
    counts, ids, corners, _ = det.detect_pose_batch(frames, K_SYN, D_ZERO, 0.14)
    counts, ids, corners = counts.copy(), ids.copy(), corners.copy().reshape(len(frames), MAXM, 8)
    boards, ch, dia = det.last_board_poses(), det.last_charuco(), det.last_diamonds()
    n_dia = 0
    for f, frame in enumerate(frames):
        n = int(counts[f])
        _check_frame(ids[f, :n], corners[f, :n].reshape(-1, 4, 2), frame, do.DICT_ID, 32, 0.02, vs_cv2=False)
        assert [bytes(r) for r in boards[f]] == [bytes(r) for r in det.board_poses(ids[f, :n], corners[f, :n], K_SYN, D_ZERO)], f
        sch = det.charuco(frame, ids[f, :n], corners[f, :n], K_SYN, D_ZERO)
        for (br, bi, bxy), (sr, si, sxy) in zip(ch[f], sch):
            assert bytes(br) == bytes(sr) and np.array_equal(bi, si) and np.array_equal(bxy, sxy), f
        si, sc, srec = det.diamonds(frame, ids[f, :n], corners[f, :n], K_SYN, D_ZERO)
        assert np.array_equal(dia[f][0], si) and np.array_equal(dia[f][1], sc) and [bytes(r) for r in dia[f][2]] == [bytes(r) for r in srec], f
        n_dia += len(si)
    assert n_dia >= 6


@pytest.mark.parametrize("enc", ["bgr8", "rgb8", "mono8"])
def test_submit_collect_two_in_flight(enc):
    W, H = 1920, 1080
    K, D = synth.camera_for(W, H)
    det = _det(W, H, 32, 0.05)
    det.set_input_encoding(enc)
    frames = _frames(W, H, 4, 500)
    conv = np.ascontiguousarray(np.stack([f[:, :, ::-1] if enc == "rgb8" else (f[:, :, 0] if enc == "mono8" else f) for f in frames]))
    a, b = conv[:2].copy(), conv[2:].copy()
    det.submit_batch(a, K, D, 0.14)
    det.submit_batch(b, K, D, 0.14)
    for src in (frames[:2], frames[2:]):
        counts, ids, corners, _ = det.collect_batch()
        for f, bgr in enumerate(src):
            _check_frame(ids[f, :counts[f]], corners[f, :counts[f]], bgr, A.DICT_6X6_250, 32, 0.05, vs_cv2=False)


def test_disable_restores_default_outputs():
    W, H = 1920, 1080
    K, D = synth.camera_for(W, H)
    frames = np.stack(_frames(W, H, 2, 600))
    plain = Detector(default_params(dictionary=A.DICT_6X6_250), max_width=W, max_height=H, max_batch=4)
    ref = [x.copy() for x in plain.detect_pose_batch(frames, K, D, 0.14)[:3]]
    ref_tf = bytes(plain.detect_pose_batch(frames, K, D, 0.14)[3])
    det = _det(W, H, 32, 0.02)
    det.detect_pose_batch(frames, K, D, 0.14)
    det.set_aruco3(enable=False)
    got = det.detect_pose_batch(frames, K, D, 0.14)
    assert ref[0].sum() >= 10
    for x, y in zip(got[:3], ref):
        assert np.array_equal(x, y)
    assert bytes(got[3]) == ref_tf


def test_refusals():
    W, H = 640, 480
    det = _det(W, H)
    bgr = _frames(W, H, 1, 700)[0]
    det.detect(bgr)
    lib = det.lib
    specs = (_lib.fid_dictionary_spec * 2)(_lib.fid_dictionary_spec(A.DICT_6X6_250, 0, 0.0), _lib.fid_dictionary_spec(A.DICT_4X4_50, 0, 0.0))
    assert lib.fid_set_dictionaries(det.h, 2, specs) == FID_ERR_UNSUPPORTED
    n = C.c_int(0)
    ids = np.zeros(MAXM, np.int32)
    corners = np.zeros((MAXM, 8), np.float32)
    assert lib.fid_detect_multi_dict(det.h, bgr.ctypes.data_as(C.c_void_p), W, H, W * 3, MAXM, C.byref(n), ids.ctypes.data_as(C.c_void_p),
                                     corners.ctypes.data_as(C.c_void_p), None) == FID_ERR_UNSUPPORTED
    assert lib.fid_set_batch_marker_refinement(det.h, 1) == FID_ERR_UNSUPPORTED
    assert lib.fid_debug_rejected(det.h, MAXM, C.byref(n), corners.ctypes.data_as(C.c_void_p)) == FID_ERR_UNSUPPORTED
    for bad in [(0, 0.02), (32, -0.1), (32, 1.5), (32, float("nan"))]:
        with pytest.raises(_lib.FidError):
            det.set_aruco3(*bad)
    # the other direction: with several dictionaries or batch refinement, the mode is refused
    other = Detector(default_params(), max_width=W, max_height=H, max_batch=1)
    other.set_dictionaries([A.DICT_6X6_250, A.DICT_4X4_50])
    with pytest.raises(_lib.FidError):
        other.set_aruco3(32, 0.02)
    det.set_aruco3(enable=False)
    assert lib.fid_set_dictionaries(det.h, 2, specs) == _lib.FID_OK
