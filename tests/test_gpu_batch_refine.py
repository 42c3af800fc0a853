"""detectMarkers' rejected list on the device (fid_debug_rejected) and refinement of missed board markers inside the batch calls
(fid_set_batch_marker_refinement, fid_last_marker_refinement) against cv2 4.13 detectMarkers + refineDetectedMarkers."""
import ctypes as C

import cv2
import numpy as np
import pytest

from fiducials_b200 import _lib
from fiducials_b200.node import MAXM, Detector, default_params
import marker_refine_oracle as mo
import rejected_cases as rc

pytestmark = pytest.mark.gpu

D_ZERO = np.zeros(5)
REFINE = (10.0, 3.0, True)
FID_MAX_BOARDS = 16


def _frames_for_rejected():
    frames = list(rc.synthetic_frames()) + list(rc.border_frames())[::3] + list(rc.nested_frames()) + list(rc.damaged_frames(6))
    rng = np.random.default_rng(0)
    frames.append(("blank", np.full((480, 640, 3), 128, np.uint8), 10))
    frames.append(("noise", rng.integers(0, 256, (480, 640, 3), dtype=np.uint8), 10))
    return frames


@pytest.mark.parametrize("method", [0, 1, 2])
def test_debug_rejected_matches_cv2(method):
    """Count, order and corners bit-identical with rejectedImgPoints, for every corner refinement method."""
    dets = {}
    n_rej = 0
    try:
        for name, bgr, d in _frames_for_rejected():
            H, W = bgr.shape[:2]
            key = (d, W, H)
            if key not in dets:
                dets[key] = Detector(default_params(dictionary=d, cornerRefinementMethod=method), 0, W, H, 1)
            det = dets[key]
            ids, _ = det.detect(bgr)
            rej = det.debug_rejected()
            rids, _, rrej = rc.cv2_lists(bgr, d, cornerRefinementMethod=method)
            assert ids.tolist() == rids.tolist(), name
            assert rej.shape == rrej.shape and np.array_equal(rej, rrej), name
            # k_finish and k_rejected each replay the candidate hierarchy: every selected candidate is in exactly one list
            assert len(ids) + len(rej) == det.last_counters()["selected"], name
            n_rej += len(rej)
    finally:
        for det in dets.values():
            det.close()
    assert n_rej > 50


def _board_frames(n, size=(5, 4)):
    board = None
    frames, grays = [], []
    for seed in range(n):
        board, g = rc.damaged_board(seed, ("near", "far", "oblique")[seed % 3], size)
        grays.append(g)
        frames.append(cv2.cvtColor(g, cv2.COLOR_GRAY2BGR))
    return board, np.ascontiguousarray(np.stack(frames)), grays


def _refine_detector(max_batch, boards=(), charuco=(), batch=True, refine=REFINE):
    det = Detector(default_params(dictionary=mo.DICT), 0, rc.W, rc.H, max_batch)
    if boards:
        det.set_boards(boards)
    if charuco:
        det.set_charuco_boards(charuco)
    det.set_marker_refinement(*refine)
    det.set_batch_marker_refinement(batch)
    return det


def _check_against_cv2(grays, boards, out, last, off, K, D, det, refine=REFINE, labels=None, method=1):
    """ids, recovered indices and boards (labels[b] for cv2's board b: b, or FID_MAX_BOARDS + c for ChArUco board c) identical to
    cv2; rejected list before refinement identical to detectMarkers'; detected markers identical to the batch without refinement;
    recovered corners within 1e-3 px of cv2; recovered poses identical to fid_pose on the device's corners.  Returns (recovered, bit-identical corners)."""
    counts, ids, corners, tfs = out
    ocounts, oids, ocorners, otfs = off
    cvdet = mo.detector(refine, cornerRefinementMethod=method)
    labels = list(range(len(boards))) if labels is None else labels
    n_rec = n_bit = 0
    for f, g in enumerate(grays):
        rids, rcorners, rrej = mo.detect(cvdet, g)
        ri, rcr, rr, rx, rb, _ = mo.refine(cvdet, g, boards, rids, rcorners, rrej, K, D)
        n, n0 = int(counts[f]), int(ocounts[f])
        idx, brd, before, left = last[f]
        assert ids[f, :n].tolist() == ri.tolist(), f
        assert idx.tolist() == rx and brd.tolist() == [labels[b] for b in rb], f
        assert np.array_equal(before, rrej) and np.array_equal(left, rr), f
        assert n == n0 + len(idx)
        assert np.array_equal(ids[f, :n0], oids[f, :n0]) and np.array_equal(corners[f, :n0], ocorners[f, :n0])
        assert np.abs(corners[f, n0:n] - rcr[n0:]).max(initial=0.0) <= 1e-3, f
        n_bit += int(sum(np.array_equal(corners[f, m], rcr[m]) for m in range(n0, n)))
        n_rec += n - n0
        if K is not None:
            for m in range(n0):
                assert bytes(tfs[f * MAXM + m]) == bytes(otfs[f * MAXM + m])
            if n > n0:
                ref = det.pose(ids[f, n0:n], corners[f, n0:n], K, D, 0.14)
                for m in range(n0, n):
                    assert bytes(tfs[f * MAXM + m]) == bytes(ref[m - n0]), (f, m)
    return n_rec, n_bit


def _copy(out):
    counts, ids, corners, tfs = out
    return counts.copy(), ids.copy(), corners.copy(), None if tfs is None else type(tfs).from_buffer_copy(tfs)


@pytest.mark.parametrize("camera", ["none", "D_zero", "D_ref"])
def test_batch_refinement_matches_cv2(camera):
    """Grid boards in a multi-chunk batch (10 frames, chunks of 4), against cv2 board after board."""
    board, frames, grays = _board_frames(10)
    K, D = (None, None) if camera == "none" else (rc.K_SYN, D_ZERO if camera == "D_zero" else rc.D_REF)
    det = _refine_detector(4, [board])
    try:
        det.set_batch_marker_refinement(False)
        off = _copy(det.detect_pose_batch(frames, K, D, 0.14))
        det.set_batch_marker_refinement(True)
        out = _copy(det.detect_pose_batch(frames, K, D, 0.14))
        last = det.last_marker_refinement()
        n_rec, n_bit = _check_against_cv2(grays, [board], out, last, off, K, D, det)
        assert n_rec >= 10
        print("\n%s: %d recovered, %d bit-identical with cv2" % (camera, n_rec, n_bit))
        # board poses of the refined lists equal fid_estimate_board_poses on them
        if K is not None:
            counts, ids, corners, _ = out
            recs = det.last_board_poses()
            for f in range(len(frames)):
                n = int(counts[f])
                ref = det.board_poses(ids[f, :n], corners[f, :n], K, D)
                assert bytes(recs[f][0]) == bytes(ref[0])
    finally:
        det.close()


@pytest.mark.parametrize("method", [0, 1])
@pytest.mark.parametrize("refine", [(3.0, 3.0, True), (40.0, 3.0, True), (10.0, -1.0, True), (10.0, 3.0, False)])
def test_batch_parameters(refine, method):
    """The refinement parameters (minRepDistance 3 / 40, no bit check, one corner order) under CORNER_REFINE_NONE and SUBPIX, with
    and without a camera."""
    board, frames, grays = _board_frames(6, (6, 5))
    det = Detector(default_params(dictionary=mo.DICT, cornerRefinementMethod=method), 0, rc.W, rc.H, 6)
    try:
        det.set_boards([board])
        det.set_marker_refinement(*refine)
        for K in (None, rc.K_SYN):
            det.set_batch_marker_refinement(False)
            off = _copy(det.detect_pose_batch(frames, K, D_ZERO, 0.14))
            det.set_batch_marker_refinement(True)
            out = _copy(det.detect_pose_batch(frames, K, D_ZERO, 0.14))
            _check_against_cv2(grays, [board], out, det.last_marker_refinement(), off, K, D_ZERO, det, refine=refine, method=method)
    finally:
        det.close()


def test_batch_refinement_in_flight_and_device_frames():
    """Two batches in flight through submit/collect, and device-resident frames, give what the synchronous call gives; the refined
    lists equal fid_refine_detected_markers on fid_debug_rejected's list."""
    import torch

    board, frames, grays = _board_frames(6)
    det = _refine_detector(3, [board])
    try:
        ref = _copy(det.detect_pose_batch(frames, rc.K_SYN, D_ZERO, 0.14))
        ref_last = det.last_marker_refinement()
        det.submit_batch(frames[:3], rc.K_SYN, D_ZERO, 0.14)
        det.submit_batch(frames[3:], rc.K_SYN, D_ZERO, 0.14)
        for part, sl in ((det.collect_batch(), slice(0, 3)), (None, slice(3, 6))):
            if part is None:
                part = det.collect_batch()
            last = det.last_marker_refinement()
            counts, ids, corners, tfs = part
            for i, f in enumerate(range(sl.start, sl.stop)):
                n = int(counts[i])
                assert n == ref[0][f] and np.array_equal(ids[i, :n], ref[1][f, :n]) and np.array_equal(corners[i, :n], ref[2][f, :n])
                assert all(bytes(tfs[i * MAXM + m]) == bytes(ref[3][f * MAXM + m]) for m in range(n))
                for a, b in zip(last[i], ref_last[f]):
                    assert np.array_equal(a, b)
        dev = torch.from_numpy(frames).cuda()
        torch.cuda.synchronize()
        out = det.detect_pose_batch(dev.data_ptr(), rc.K_SYN, D_ZERO, 0.14, on_device=True, n_frames=len(frames), width=rc.W, height=rc.H)
        assert np.array_equal(out[0], ref[0]) and np.array_equal(out[1], ref[1]) and np.array_equal(out[2], ref[2])
        # the one-frame call on the device's own rejected list
        for f in range(len(frames)):
            ids0, corners0 = det.detect(frames[f])
            rej = det.debug_rejected()
            gi, gc, left, gx, gb = det.refine_markers(frames[f], ids0, corners0, rej, rc.K_SYN, D_ZERO)
            n = int(ref[0][f])
            assert gi.tolist() == ref[1][f, :n].tolist() and np.array_equal(gc, ref[2][f, :n])
            assert gx.tolist() == ref_last[f][0].tolist() and np.array_equal(left, ref_last[f][3])
    finally:
        det.close()


def test_grid_and_charuco_together():
    """A grid board and a ChArUco board set together, both in every frame with damaged markers: refinement runs the grid, then the
    ChArUco board (label FID_MAX_BOARDS), as cv2 does board after board, and k_charuco sees the refined lists: its records change
    and equal fid_detect_charuco on those lists."""
    scenes = [rc.grid_and_charuco(seed) for seed in range(6)]
    grid, ch = scenes[0][0], scenes[0][1]
    grays = [g for _, _, g in scenes]
    frames = np.ascontiguousarray(np.stack([cv2.cvtColor(g, cv2.COLOR_GRAY2BGR) for g in grays]))
    det = _refine_detector(4, [grid], [ch])
    try:
        for K in (None, rc.K_SYN):
            det.set_batch_marker_refinement(False)
            off = _copy(det.detect_pose_batch(frames, K, D_ZERO, 0.14))
            off_ch = det.last_charuco()
            det.set_batch_marker_refinement(True)
            out = _copy(det.detect_pose_batch(frames, K, D_ZERO, 0.14))
            last = det.last_marker_refinement()
            n_rec, _ = _check_against_cv2(grays, [grid, ch], out, last, off, K, D_ZERO, det, labels=[0, FID_MAX_BOARDS])
            labels = [b for r in last for b in r[1].tolist()]
            assert 0 in labels and FID_MAX_BOARDS in labels, labels
            recs = det.last_charuco()
            counts, ids, corners, _ = out
            changed = 0
            for f in range(len(frames)):
                n = int(counts[f])
                ref = det.charuco(frames[f], ids[f, :n], corners[f, :n], K, D_ZERO)
                assert bytes(recs[f][0][0]) == bytes(ref[0][0])
                assert np.array_equal(recs[f][0][1], ref[0][1]) and np.array_equal(recs[f][0][2], ref[0][2])
                changed += recs[f][0][0].n_corners != off_ch[f][0][0].n_corners
            assert changed > 0
    finally:
        det.close()


def _launches(det):
    return det.last_counters()["kernel_launches"]


def test_off_means_off():
    """Never set, set and cleared, set without boards, or without fid_set_marker_refinement: the same bytes and launches as a
    handle that never heard of it."""
    board, frames, _ = _board_frames(5)
    base = Detector(default_params(dictionary=mo.DICT), 0, rc.W, rc.H, 5)
    base.set_boards([board])
    ref = _copy(base.detect_pose_batch(frames, rc.K_SYN, D_ZERO, 0.14))
    ref_launch = _launches(base)
    base.close()
    variants = []
    d1 = _refine_detector(5, [board], batch=True)
    d1.set_batch_marker_refinement(False)
    variants.append(d1)
    d2 = Detector(default_params(dictionary=mo.DICT), 0, rc.W, rc.H, 5)
    d2.set_marker_refinement(*REFINE)
    d2.set_batch_marker_refinement(True)
    variants.append(d2)  # no board: compare without boards below
    d3 = Detector(default_params(dictionary=mo.DICT), 0, rc.W, rc.H, 5)
    d3.set_boards([board])
    d3.set_batch_marker_refinement(True)
    variants.append(d3)  # batch switch without refinement parameters
    try:
        for i, det in enumerate(variants):
            if i == 1:
                nob = Detector(default_params(dictionary=mo.DICT), 0, rc.W, rc.H, 5)
                r = _copy(nob.detect_pose_batch(frames, rc.K_SYN, D_ZERO, 0.14))
                rl = _launches(nob)
                nob.close()
            else:
                r, rl = ref, ref_launch
            out = det.detect_pose_batch(frames, rc.K_SYN, D_ZERO, 0.14)
            assert _launches(det) == rl, i
            for a, b in zip(out[:3], r[:3]):
                assert np.array_equal(a, b), i
            assert bytes(out[3]) == bytes(r[3]), i
            with pytest.raises(_lib.FidError):
                det.last_marker_refinement()
    finally:
        for det in variants:
            det.close()


def _full_frames():
    """Two 1080p frames of a 20 x 13 GridBoard of DICT_5X5_1000 (260 markers) with the inner bits of 4 and 8 markers painted white:
    detection finds 256 and 252 markers, the FID_MAX_MARKERS limit and four below it.  Also cv2's detected lists and recovered ids
    (RefineParameters(10, -1, true), no camera)."""
    from oracle import aruco_oracle as ao

    d = cv2.aruco.getPredefinedDictionary(7)
    gb = cv2.aruco.GridBoard((20, 13), 64, 12, d)
    clean = np.full((1080, 1920), 128, np.uint8)
    clean[12:1068, 166:1754] = gb.generateImage((1588, 1056), marginSize=40, borderBits=1)
    cvdet = cv2.aruco.ArucoDetector(d, ao.reference_detector_params(), cv2.aruco.RefineParameters(10, -1, True))
    c, ids, _ = cvdet.detectMarkers(clean)
    pos = {int(i): q.reshape(4, 2) for i, q in zip(ids.reshape(-1), c)}
    frames, expect = [], []
    for n in (4, 8):
        g = clean.copy()
        for k in np.random.default_rng(n).choice(260, n, replace=False):
            (x0, y0), (x1, y1) = pos[int(k)].min(0), pos[int(k)].max(0)
            dx, dy = (x1 - x0) / 7, (y1 - y0) / 7
            g[int(round(y0 + dy)):int(round(y1 - dy)), int(round(x0 + dx)):int(round(x1 - dx))] = 255
        c, ids, rej = cvdet.detectMarkers(g)
        c2, i2, _, _ = cvdet.refineDetectedMarkers(g, gb, c, ids, rej)
        frames.append(cv2.cvtColor(g, cv2.COLOR_GRAY2BGR))
        expect.append((ids.reshape(-1).tolist(), i2.reshape(-1)[len(ids):].tolist()))
    return np.ascontiguousarray(np.stack(frames)), expect


def test_max_markers_overflow():
    """A recovered marker that finds no slot below FID_MAX_MARKERS: the batch returns FID_ERR_CAPACITY, that frame stops refining
    there (a frame already at the limit recovers nothing, one four below keeps cv2's first four), and fid_last_marker_refinement
    describes what was produced."""
    from fiducials_b200.board import grid_board

    frames, expect = _full_frames()
    assert [len(e[0]) for e in expect] == [256, 252] and all(len(e[1]) >= 4 for e in expect)
    det = Detector(default_params(dictionary=7), 0, 1920, 1080, 2)
    try:
        det.set_boards([grid_board((20, 13), 64, 12)])
        det.set_marker_refinement(10.0, -1.0, True)
        off = _copy(det.detect_pose_batch(frames))
        assert off[0].tolist() == [256, 252]
        det.set_batch_marker_refinement(True)
        with pytest.raises(_lib.FidError) as e:
            det.detect_pose_batch(frames)
        assert e.value.status == -5
        counts, ids, _, _ = det._out  # the wrapper's output buffers, written before the status was returned
        last = det.last_marker_refinement()
        assert counts.tolist() == [256, 256]
        assert len(last[0][0]) == 0 and len(last[1][0]) == 4
        assert ids[0, :256].tolist() == expect[0][0]
        assert ids[1, :256].tolist() == expect[1][0] + expect[1][1][:4]
        assert len(last[0][2]) == 4 and len(last[1][2]) == 8  # the painted markers are the rejected candidates
    finally:
        det.close()


def test_errors():
    scenes = [rc.grid_and_charuco(seed) for seed in range(2)]  # three markers recovered in each
    frames = np.ascontiguousarray(np.stack([cv2.cvtColor(g, cv2.COLOR_GRAY2BGR) for _, _, g in scenes]))
    det = _refine_detector(2, [scenes[0][0]], [scenes[0][1]])
    lib, h = det.lib, det.h
    try:
        det.submit_batch(frames, rc.K_SYN, D_ZERO, 0.14)
        assert lib.fid_set_batch_marker_refinement(h, 0) == -1  # batches in flight
        det.collect_batch()
        nf = C.c_int(0)
        nrec = np.zeros(2, np.int32)
        nrej = np.zeros(2, np.int32)
        assert lib.fid_last_marker_refinement(h, 0, 0, C.byref(nf), nrec.ctypes.data_as(C.c_void_p), None, None, nrej.ctypes.data_as(C.c_void_p), None) == 0
        assert nf.value == 2 and nrec.sum() > 0 and nrej.sum() > 0
        assert nrej.max() > 1 and nrec.max() > 1  # the capacity cases below need a frame with two of each
        small = np.zeros((2, 1, 8), np.float32)
        nf.value = -7  # a rejected buffer too small: FID_ERR_CAPACITY, nothing written
        assert lib.fid_last_marker_refinement(h, 0, 1, C.byref(nf), None, None, None, None, small.ctypes.data_as(C.c_void_p)) == -5
        assert not small.any() and nf.value == -7
        ri = np.zeros((2, 1), np.int32)
        assert lib.fid_last_marker_refinement(h, 1, 0, C.byref(nf), None, ri.ctypes.data_as(C.c_void_p), None, None, None) == -5
        assert not ri.any() and nf.value == -7
        det.set_batch_marker_refinement(False)
        det.detect_pose_batch(frames, rc.K_SYN, D_ZERO, 0.14)
        assert lib.fid_last_marker_refinement(h, 0, 0, C.byref(nf), None, None, None, None, None) == -1  # that batch did not refine
        fresh = Detector(default_params(dictionary=mo.DICT), 0, rc.W, rc.H, 1)
        try:  # no fid_detect yet: no candidate lists to gather from
            assert fresh.lib.fid_debug_rejected(fresh.h, 16, C.byref(nf), None) == -1
        finally:
            fresh.close()
    finally:
        det.close()


def test_node_refine_markers():
    """FiducialsNode(boards=[...], refine_markers=...): process_batch (with the camera) and the per-frame callbacks (imageCallback
    refines without one) report the recovered markers like any other marker and carry `.recovered`; ignore_fiducials applies to
    them."""
    from fiducials_b200.node import FiducialsNode

    board, frames, grays = _board_frames(3)
    cvdet = mo.detector(REFINE)
    expect = {}
    for K in (None, rc.K_SYN):
        expect[K is None] = []
        for g in grays:
            rids, rcorners, rrej = mo.detect(cvdet, g)
            ri = mo.refine(cvdet, g, [board], rids, rcorners, rrej, K, D_ZERO)[0]
            expect[K is None].append((ri.tolist(), ri[len(rids):].tolist()))
    ignored = expect[False][0][1][0]
    with pytest.raises(ValueError):
        FiducialsNode(dictionary=mo.DICT, refine_markers=REFINE, max_width=rc.W, max_height=rc.H)
    node = FiducialsNode(dictionary=mo.DICT, boards=[board], refine_markers=REFINE, ignore_fiducials=[ignored], max_width=rc.W, max_height=rc.H,
                         max_batch=3)
    node.camInfoCallback(rc.K_SYN, D_ZERO)
    res = node.process_batch(frames)
    kept = lambda ids: [i for i in ids if i != ignored]
    for f in range(len(frames)):
        ids, rec = expect[False][f]
        assert [t.fiducial_id for t in res[f].transforms] == kept(ids)
        assert [i for i, _ in res[f].recovered] == kept(rec)
        ids, rec = expect[True][f]
        fva = node.imageCallback(frames[f])
        assert [x.fiducial_id for x in fva.fiducials] == kept(ids)
        assert [i for i, _ in fva.recovered] == kept(rec)
        fta = node.poseEstimateCallback(fva)
        assert [t.fiducial_id for t in fta.transforms] == kept(ids)
        assert fta.recovered == fva.recovered
