"""ChArUco diamonds on the device (fid_set_diamonds, fid_detect_diamonds, fid_last_diamonds) against the host build of the same
arithmetic (diamond.cuh) and cv2's CharucoDetector.detectDiamonds + solvePnP, and every other output with diamonds on and off."""
import ctypes as C

import cv2
import numpy as np
import pytest

from fiducials_b200 import _lib
from fiducials_b200.board import charuco_board, grid_board
from fiducials_b200.node import MAXM, Detector, FiducialsNode, default_params
import diamond_oracle as do
from test_hostsim_diamond import D_REF, D_ZERO, H, K_SYN, RATIOS, W, check, hs_diamonds, scene

pytestmark = pytest.mark.gpu

FLEN = 0.14
SQ, MK = RATIOS[0]


def _frames(n, seed, ratio=RATIOS[0]):
    """n BGR frames with 1 to 4 diamonds each (some with a marker covered, stray markers, close together); every 4th frame blank."""
    rng = np.random.default_rng(seed)
    out = []
    for f in range(n):
        if f % 4 == 3:
            g = np.full((H, W), 128, np.uint8)
        else:
            kind = ["near", "far", "oblique"][f % 3]
            nd = 1 if kind == "near" else int(rng.integers(2, 5))
            g, _ = scene(rng, nd, kind, ratio, cover=int(rng.integers(0, 2)), strays=int(rng.integers(0, 3)), close=f % 2 == 1 and nd > 1)
        out.append(cv2.cvtColor(g, cv2.COLOR_GRAY2BGR))
    return np.ascontiguousarray(np.stack(out))


def _assert_matches_host(recs, gray, ids, corners, K, D, what):
    """Device records against the host build: identical ids and order, bit-identical corners, poses within 1e-8 (the device's
    double sin / cos / exp differ from the host C library's in the last bit for some arguments, and the LM trajectory carries it)."""
    hi, hc, hp = hs_diamonds(gray, ids, corners, SQ, MK, K, D)
    assert [list(r.ids) for r in recs] == hi.tolist(), what
    assert np.array_equal(np.array([list(r.corners) for r in recs], np.float32).reshape(-1, 4, 2), hc), what
    for r, p in zip(recs, hp):
        assert r.status == int(p[0]) and r.pose.fiducial_id == r.ids[0], what
        if r.status == 1:
            assert np.abs(np.array(list(r.pose.rvec)) - p[1:4]).max() <= 1e-8 and np.abs(np.array(list(r.pose.translation)) - p[4:7]).max() <= 1e-8, what
            assert np.abs(np.array(list(r.pose.rotation)) - p[7:11]).max() <= 1e-8, what
    return len(recs)


@pytest.mark.parametrize("camera", ["none", "D_zero", "D_ref"])
def test_detect_diamonds_matches_host_and_cv2(camera):
    K, D = (None, None) if camera == "none" else (K_SYN, D_ZERO if camera == "D_zero" else D_REF)
    frames = _frames(12, 1)
    det = Detector(default_params(dictionary=do.DICT_ID), 0, W, H, 2)
    det.set_diamonds(SQ, MK)
    total = 0
    for f, frame in enumerate(frames):
        counts, ids, corners, _ = det.detect_pose_batch(frame[None])
        n = int(counts[0])
        ids, corners = ids[0, :n], corners.reshape(1, MAXM, 8)[0, :n].reshape(-1, 4, 2)
        gray = cv2.cvtColor(frame, cv2.COLOR_BGR2GRAY)
        di, dc, recs = det.diamonds(frame, ids, corners, K, D)
        total += _assert_matches_host(recs, gray, ids, corners, K, D, "frame %d" % f)
        assert np.array_equal(di, np.array([list(r.ids) for r in recs], np.int32).reshape(-1, 4))
        if n:
            check(gray, ids, corners, SQ, MK, K, D, what="device frame %d" % f)  # the host build against cv2 on the device's markers
        if f % 4 == 3:
            assert len(recs) == 0
    assert total >= 6, total
    det.close()


def test_batches_match_single_frame_calls_and_other_outputs_unchanged():
    """Multi-chunk batches with diamonds on and off: every other output byte for byte, the same kernel launches when off, and per
    frame the single-frame call on the batch's own markers, bit for bit."""
    frames = _frames(9, 2)
    det = Detector(default_params(dictionary=do.DICT_ID), 0, W, H, 4)  # 3 chunks per 9-frame batch
    det.set_pose_hypotheses(True)
    res, launches = [], []
    for on in (False, True, False):
        det.set_diamonds(SQ if on else None, MK)
        det.submit_batch(frames, K_SYN, D_ZERO, FLEN)
        counts, ids, corners, tfs = det.collect_batch()
        res.append((counts.tobytes(), ids.tobytes(), corners.tobytes(), bytes(tfs), bytes(det.last_pose_hypotheses())))
        launches.append(det.last_counters()["kernel_launches"])
        if not on:
            with pytest.raises(_lib.FidError):
                det.last_diamonds()
            continue
        dia = det.last_diamonds()
        assert len(dia) == len(frames)
        corners = corners.reshape(len(frames), MAXM, 8)
        for f in range(len(frames)):
            n = int(counts[f])
            si, sc, srec = det.diamonds(frames[f], ids[f, :n], corners[f, :n], K_SYN, D_ZERO)
            bi, bc, brec = dia[f]
            assert np.array_equal(bi, si) and np.array_equal(bc, sc) and [bytes(r) for r in brec] == [bytes(r) for r in srec], f
        assert sum(len(d[0]) for d in dia) >= 5
    assert res[0] == res[1] == res[2]
    assert launches[0] == launches[2] and launches[1] == launches[0] + 3  # one k_diamond per chunk
    # no camera: diamonds without a pose
    det.set_diamonds(SQ, MK)
    counts, ids, corners, _ = det.detect_pose_batch(frames)
    dia = det.last_diamonds()
    assert sum(len(d[0]) for d in dia) > 0 and all(r.status == 0 for d in dia for r in d[2])
    det.close()


def test_with_batch_refinement_and_charuco_boards():
    """Diamonds read each frame's final markers: those batch refinement recovers included, next to a ChArUco board stage."""
    frames = _frames(6, 3)
    det = Detector(default_params(dictionary=do.DICT_ID), 0, W, H, 4)
    det.set_charuco_boards([charuco_board((5, 4), 0.03, 0.022)])
    det.set_boards([grid_board((2, 2), 0.03, 0.008, [240, 241, 242, 243])])
    det.set_marker_refinement(10.0, 3.0, True)
    det.set_batch_marker_refinement(True)
    det.set_diamonds(SQ, MK)
    counts, ids, corners, _ = det.detect_pose_batch(frames, K_SYN, D_ZERO, FLEN)
    dia = det.last_diamonds()
    ch = det.last_charuco()
    assert len(ch) == len(dia) == len(frames)
    corners = corners.reshape(len(frames), MAXM, 8)
    for f in range(len(frames)):
        n = int(counts[f])
        si, sc, srec = det.diamonds(frames[f], ids[f, :n], corners[f, :n], K_SYN, D_ZERO)
        assert np.array_equal(dia[f][0], si) and np.array_equal(dia[f][1], sc), f
        gray = cv2.cvtColor(frames[f], cv2.COLOR_BGR2GRAY)
        _assert_matches_host(srec, gray, ids[f, :n], corners[f, :n].reshape(-1, 4, 2), K_SYN, D_ZERO, "refined frame %d" % f)
    det.close()


def test_errors():
    det = Detector(default_params(dictionary=do.DICT_ID), 0, W, H, 2)
    lib = det.lib
    frame = np.zeros((480, 640, 3), np.uint8)

    def set_raw(**kw):
        p = _lib.fid_diamond_params()
        p.enable, p.square_length, p.marker_length, p.min_markers, p.check_markers = 1, 0.04, 0.03, 2, 1
        for k, v in kw.items():
            setattr(p, k, v)
        return lib.fid_set_diamonds(det.h, C.byref(p))

    assert set_raw(marker_length=0.04) == -1 and set_raw(marker_length=0.0) == -1 and set_raw(square_length=float("nan")) == -1
    assert set_raw(square_length=float("inf")) == -1 and set_raw(min_markers=3) == -1 and set_raw(min_markers=-1) == -1
    assert lib.fid_set_diamonds(det.h, None) == -1
    nd, nf = C.c_int(-1), C.c_int(0)
    out = (_lib.fid_diamond * _lib.FID_MAX_DIAMONDS)()
    args = (frame.ctypes.data_as(C.c_void_p), 640, 480, 640 * 3, 0, None, None, None, C.byref(nd), C.cast(out, C.c_void_p))
    assert lib.fid_detect_diamonds(det.h, *args) == -1  # off
    assert lib.fid_last_diamonds(det.h, 4, C.byref(nf), None, None) == -1
    assert set_raw() == 0
    assert lib.fid_detect_diamonds(det.h, *args) == 0 and nd.value == 0
    frames = _frames(3, 4)
    det.submit_batch(frames)
    assert set_raw() == -1 and lib.fid_detect_diamonds(det.h, *args) == -1  # not while a batch is in flight
    det.collect_batch()
    counts = np.zeros(3, np.int32)
    assert lib.fid_last_diamonds(det.h, 0, C.byref(nf), counts.ctypes.data_as(C.c_void_p), None) == 0 and nf.value == 3
    m = int(counts.max())
    assert m >= 1, counts
    big = (_lib.fid_diamond * (3 * m))()
    assert lib.fid_last_diamonds(det.h, m - 1, C.byref(nf), None, C.cast(big, C.c_void_p)) == -5  # FID_ERR_CAPACITY
    assert all(bytes(r) == bytes(_lib.fid_diamond()) for r in big)  # nothing written
    assert lib.fid_last_diamonds(det.h, m, C.byref(nf), None, C.cast(big, C.c_void_p)) == 0
    assert set_raw(enable=0) == 0  # off again
    det.close()


def test_node_attaches_diamonds():
    frames = _frames(3, 6)
    plain = FiducialsNode(dictionary=do.DICT_ID, fiducial_len=FLEN, max_width=W, max_height=H, max_batch=2)
    node = FiducialsNode(dictionary=do.DICT_ID, fiducial_len=FLEN, max_width=W, max_height=H, max_batch=2, diamonds=(SQ, MK))
    for nd in (plain, node):
        nd.camInfoCallback(K_SYN, D_ZERO, "camera")
    fta0 = plain.poseEstimateCallback(plain.imageCallback(frames[0]))
    fta = node.poseEstimateCallback(node.imageCallback(frames[0]))
    assert fta.transforms == fta0.transforms and not hasattr(fta0, "diamonds")
    ids, corners, recs = fta.diamonds
    assert len(ids) >= 1 and all(r.status == 1 for r in recs)
    batch0, batch = plain.process_batch(frames), node.process_batch(frames)
    for x, y in zip(batch0, batch):
        assert x.transforms == y.transforms and hasattr(y, "diamonds")
    assert np.array_equal(batch[0].diamonds[0], ids) and np.array_equal(batch[0].diamonds[1], corners)
    for n in (plain, node):
        n.det.close()
