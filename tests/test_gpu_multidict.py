"""Detection with several dictionaries on the device (fid_set_dictionaries, fid_detect_multi_dict, the batch calls): against cv2's
detectMarkersMultiDict and, bit for bit, against the host chain (tests/hostsim/multidict_hostsim.cpp); published ids and lengths
against fid_pose; the argument and mode rules."""
import ctypes as C

import numpy as np
import pytest

from fiducials_b200 import _lib, synth
from fiducials_b200.node import Detector, FiducialSlam, default_params
import multidict_oracle as mo

pytestmark = pytest.mark.gpu
A = mo.A
W, H = 1920, 1080
K, D = synth.camera_for(W, H)
DL = mo.DICT_LISTS["four"]


def _frames(n, dl=DL, seed=0):
    return [mo.render_mixed(W, H, dl, seed + i, n_markers=20) for i in range(n)]


def _det(dl=DL, method=1, max_batch=4, specs=None):
    d = Detector(default_params(cornerRefinementMethod=method, dictionary=dl[0]), max_width=W, max_height=H, max_batch=max_batch)
    d.set_dictionaries(specs if specs is not None else [(x, 0, 0.0) for x in dl])
    return d


@pytest.mark.parametrize("method", [0, 1, 2])
def test_single_frame_matches_host_and_cv2(method):
    det = _det(method=method)
    for i, bgr in enumerate(_frames(2, seed=10 * method)):
        ids, corners, di = det.detect_multi_dict(bgr)
        hids, hcorners, hdi = mo.host_multi(bgr, DL, method)
        assert ids.tolist() == hids.tolist() and di.tolist() == hdi.tolist(), i
        if method == 2:
            assert np.abs(corners - hcorners).max(initial=0) <= 1e-3
        else:
            assert np.array_equal(corners, hcorners), np.abs(corners - hcorners).max(initial=0)
        rids, rcorners, rdi, _ = mo.cv2_multi(bgr, DL, method)
        assert ids.tolist() == rids.tolist() and di.tolist() == rdi.tolist()
        assert len(set(di.tolist())) >= 3
        # detectMarkers stays dictionary 0 alone
        sids, _ = det.detect(bgr)
        assert sids.tolist() == ids[di == 0].tolist()


def _check_batch(det, frames, counts, ids, corners, tfs, specs, fiducial_len, overrides=None, di_all=None):
    di_all = det.last_dict_indices() if di_all is None else di_all
    for f, bgr in enumerate(frames):
        n = counts[f]
        hids, hcorners, hdi = mo.host_multi(bgr, [s[0] for s in specs], 1)
        assert ids[f, :n].tolist() == hids.tolist() and di_all[f, :n].tolist() == hdi.tolist()
        assert np.array_equal(corners[f, :n], hcorners)
        if tfs is None:
            continue
        for d, (_, off, ln) in enumerate(specs):
            sel = np.where(hdi == d)[0]
            if not len(sel):
                continue
            ref = det.pose(hids[sel] + off, hcorners[sel], K, D, ln if ln > 0 else fiducial_len, overrides)
            for j, m in enumerate(sel):
                assert bytes(tfs[f * _lib.FID_MAX_MARKERS + m]) == bytes(ref[j]), (f, d, m)


def test_batch_published_ids_and_lengths():
    specs = [(A.DICT_6X6_250, 0, 0.0), (A.DICT_APRILTAG_36h11, 1000, 0.2), (A.DICT_4X4_50, 2000, 0.0), (A.DICT_5X5_1000, 5000, 0.05)]
    det = _det(specs=specs)
    frames = np.stack(_frames(3, seed=40))
    overrides = {1003: 0.31, 3: 0.11}
    counts, ids, corners, tfs = det.detect_pose_batch(frames, K, D, 0.14, overrides)
    _check_batch(det, frames, counts, ids, corners.reshape(len(frames), -1, 4, 2), tfs, specs, 0.14, overrides)


@pytest.mark.parametrize("enc", ["rgb8", "mono8"])
def test_submit_collect_two_in_flight(enc):
    specs = [(A.DICT_6X6_250, 0, 0.0), (A.DICT_APRILTAG_36h11, 100, 0.0), (A.DICT_4X4_50, 0, 0.0), (A.DICT_5X5_1000, 7, 0.1)]
    det = _det(specs=specs)
    det.set_input_encoding(enc)
    frames = _frames(4, seed=70)
    conv = np.stack([f[:, :, ::-1] if enc == "rgb8" else f[:, :, 0] for f in frames])
    conv = np.ascontiguousarray(conv)
    a, b = conv[:2].copy(), conv[2:].copy()
    det.submit_batch(a, K, D, 0.14)
    det.submit_batch(b, K, D, 0.14)
    got = []
    for src in (frames[:2], frames[2:]):  # fid_last_dict_indices is the batch collected last; fid_pose waits for both
        got.append((src, det.collect_batch(), det.last_dict_indices()))
    for src, (counts, ids, corners, tfs), di in got:
        _check_batch(det, src, counts, ids, corners, tfs, specs, 0.14, di_all=di)


def test_device_resident_frames():
    import torch

    det = _det()
    frames = np.stack(_frames(2, seed=90))
    t = torch.from_numpy(frames).cuda()
    counts, ids, corners, _ = det.detect_pose_batch(t.data_ptr(), on_device=True, n_frames=2, width=W, height=H)
    counts, ids, corners = counts.copy(), ids.copy(), corners.copy()
    h_counts, h_ids, h_corners, _ = det.detect_pose_batch(frames)
    assert counts.tolist() == h_counts.tolist() and np.array_equal(ids, h_ids) and np.array_equal(corners, h_corners)


def test_pose_hypotheses_agree():
    specs = [(A.DICT_6X6_250, 0, 0.0), (A.DICT_APRILTAG_36h11, 1000, 0.2)]
    dl = [s[0] for s in specs]
    det = _det(dl=dl, specs=specs)
    det.set_pose_hypotheses(True)
    frames = np.stack(_frames(2, dl=dl, seed=120))
    counts, ids, corners, tfs = det.detect_pose_batch(frames, K, D, 0.14)
    hyp = det.last_pose_hypotheses()
    di = det.last_dict_indices()
    for f in range(len(frames)):
        for d, (_, off, ln) in enumerate(specs):
            sel = np.where(di[f, :counts[f]] == d)[0]
            if not len(sel):
                continue
            ref = det.pose_hypotheses(ids[f, sel] + off, corners[f, sel], K, D, ln if ln > 0 else 0.14)
            for j, m in enumerate(sel):
                assert bytes(hyp[f * _lib.FID_MAX_MARKERS + m]) == bytes(ref[j])


def test_one_entry_is_byte_identical():
    frames = np.stack(_frames(3, dl=[A.DICT_5X5_1000], seed=150))
    plain = Detector(default_params(dictionary=A.DICT_5X5_1000), max_width=W, max_height=H, max_batch=4)
    one = _det(dl=[A.DICT_5X5_1000])
    r1 = plain.detect_pose_batch(frames, K, D, 0.14)
    r1 = tuple(x.copy() if isinstance(x, np.ndarray) else bytes(x) for x in r1)
    r2 = one.detect_pose_batch(frames, K, D, 0.14)
    r2 = tuple(x.copy() if isinstance(x, np.ndarray) else bytes(x) for x in r2)
    for x, y in zip(r1, r2):
        assert (np.array_equal(x, y) if isinstance(x, np.ndarray) else x == y)
    assert int(r1[0].sum()) > 0
    assert not one.last_dict_indices().any()


def test_set_params_keeps_other_entries():
    det = _det()
    det.set_params(default_params(dictionary=A.DICT_ARUCO_ORIGINAL))
    bgr = _frames(1, dl=[A.DICT_ARUCO_ORIGINAL] + DL[1:], seed=170)[0]
    ids, _, di = det.detect_multi_dict(bgr)
    rids, _, rdi, _ = mo.cv2_multi(bgr, [A.DICT_ARUCO_ORIGINAL] + DL[1:], 1)
    assert ids.tolist() == rids.tolist() and di.tolist() == rdi.tolist()


def _raw_set(det, specs):
    arr = (_lib.fid_dictionary_spec * max(len(specs), 1))(*[_lib.fid_dictionary_spec(*s) for s in specs])
    return det.lib.fid_set_dictionaries(det.h, len(specs), C.cast(arr, C.c_void_p))


def test_argument_validation_leaves_handle_unchanged():
    det = _det(dl=DL[:2])
    bgr = _frames(1, seed=190)[0]
    before = det.detect_multi_dict(bgr)
    assert _raw_set(det, []) == -1  # n = 0
    assert _raw_set(det, [(A.DICT_4X4_50, 0, 0.0)] * 9) == -1
    assert _raw_set(det, [(A.DICT_4X4_50, 0, 0.0), (12345, 0, 0.0)]) == -4
    assert _raw_set(det, [(A.DICT_4X4_50, 0, 0.0), (A.DICT_4X4_50, 2**31 - 10, 0.0)]) == -1
    assert _raw_set(det, [(A.DICT_4X4_50, 0, -1.0)]) == -1
    after = det.detect_multi_dict(bgr)
    for x, y in zip(before, after):
        assert np.array_equal(x, y)


def _batch_bytes(det, frames):
    counts, ids, corners, tfs = det.detect_pose_batch(frames, K, D, 0.14)
    return counts.tobytes() + ids.tobytes() + corners.tobytes() + bytes(tfs) + det.last_dict_indices().tobytes()


def test_refused_combinations():
    """Boards, ChArUco boards, batch refinement and diamonds are refused with several dictionaries, in both directions, and the refused
    call changes nothing: the handle's batch outputs stay byte-identical and its switches off."""
    from fiducials_b200.board import charuco_board, grid_board

    det = _det(dl=DL[:2])
    frames = np.stack(_frames(2, seed=200))
    before = _batch_bytes(det, frames)
    board = grid_board((2, 2), 0.04, 0.01)
    for call in (lambda: det.set_boards([board]), lambda: det.set_charuco_boards([charuco_board((3, 3), 0.04, 0.03)]),
                 lambda: det.set_diamonds(0.04, 0.02)):
        with pytest.raises(_lib.FidError) as e:
            call()
        assert e.value.status == -4
    assert det.lib.fid_set_batch_marker_refinement(det.h, 1) == -4
    n_frames, n_boards = C.c_int(0), C.c_int(0)
    assert det.lib.fid_last_board_poses(det.h, 16, C.byref(n_frames), C.byref(n_boards), None) == -1  # no board was set
    assert _batch_bytes(det, frames) == before
    det.detect_multi_dict(frames[0])
    n = C.c_int(0)
    assert det.lib.fid_debug_rejected(det.h, 0, C.byref(n), None) == -4  # the multi-dictionary rejected list (finding 15)
    # the other direction: a board set first refuses a second dictionary, and the handle stays single-dictionary
    one = Detector(default_params(), max_width=W, max_height=H, max_batch=4)
    one.set_boards([board])
    ref = _batch_bytes(one, frames)
    assert _raw_set(one, [(7, 0, 0.0), (A.DICT_4X4_50, 0, 0.0)]) == -4
    assert _batch_bytes(one, frames) == ref
    one.set_boards([])
    one.set_diamonds(0.04, 0.02)
    assert _raw_set(one, [(7, 0, 0.0), (A.DICT_4X4_50, 0, 0.0)]) == -4
    assert _raw_set(one, [(7, 0, 0.0)]) == 0  # one plain entry is not multi-dictionary mode


def test_slam_keeps_offset_families_apart():
    """Two families with equal raw ids and different offsets are two landmarks in the map."""
    specs = [(A.DICT_6X6_250, 0, 0.0), (A.DICT_APRILTAG_36h11, 1000, 0.0)]
    det = _det(dl=[s[0] for s in specs], specs=specs)
    g = np.full((H, W), 200, np.uint8)
    g[300:560, 300:560] = A.generateImageMarker(A.getPredefinedDictionary(specs[0][0]), 5, 260, borderBits=1)
    g[300:560, 1200:1460] = A.generateImageMarker(A.getPredefinedDictionary(specs[1][0]), 5, 260, borderBits=1)
    frames = np.ascontiguousarray(np.stack([np.repeat(g[:, :, None], 3, axis=2)]))
    counts, ids, _, tfs = det.detect_pose_batch(frames, K, D, 0.14)
    assert ids[0, :counts[0]].tolist() == [5, 5]
    pub = [tfs[m].fiducial_id for m in range(counts[0])]
    assert pub == [5, 1005]
    from fiducials_b200.msgs import FiducialTransformArray
    from fiducials_b200.node import _to_msg

    msg = FiducialTransformArray(transforms=[_to_msg(tfs[m]) for m in range(counts[0])])
    slam = FiducialSlam()
    ident = [0, 0, 0, 0, 0, 0, 1]
    for _ in range(13):  # as smoke(): the map's first fiducial, then the robot pose, then the second
        slam.transformCallback(msg, ident, ident)
    assert sorted(int(e.fiducial_id) for e in slam.entries()) == [5, 1005]
