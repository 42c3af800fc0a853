"""Boards bound to dictionary families on the device (fid_set_family_boards, fid_set_family_charuco_boards, fid_set_family_diamonds)
in multi-dictionary batches: against cv2's composition (tests/multidict_boards_cases.py), bit for bit against the stand-alone calls
of a single-dictionary handle of each family fed corners[di == k], the single-dictionary equivalence of index 0, the argument rules
and the node."""
import ctypes as C

import numpy as np
import pytest

import board_oracle as bo
import charuco_oracle as co
import diamond_oracle as dio
import multidict_boards_cases as mc
from fiducials_b200 import _lib, synth
from fiducials_b200.node import Detector, FiducialsNode, default_params

pytestmark = pytest.mark.gpu
A = mc.A
W, H = mc.W, mc.H
K, D = synth.camera_for(W, H)
MAXM = _lib.FID_MAX_MARKERS
GRIDS = [A.DICT_4X4_50, A.DICT_5X5_1000]
MIXED = [A.DICT_6X6_250, A.DICT_APRILTAG_36h11, A.DICT_4X4_50]
OFFSETS = [0, 1000, 2000, 3000]


def _specs(dicts):
    return [(d, OFFSETS[k], 0.0) for k, d in enumerate(dicts)]


# name: (dictionary list, renderer, [(marker board, family)], [(ChArUco board, family)], diamond family or None)
CASES = {
    "grids_2": (GRIDS, mc.render_grids, [(mc.grid(), 0), (mc.grid(), 1)], [], None),
    "mixed_3": (MIXED, mc.render_mixed_boards, [(mc.grid(), 2), (mc.tags(), 1)], [(mc.charuco(), 0)], 0),
    "mixed_3_diamonds_in_36h11": (MIXED, mc.render_mixed_boards, [], [(mc.charuco(), 0)], 1),
    "listed_twice": ([A.DICT_4X4_50, A.DICT_4X4_50], lambda s: mc.render_grids(s, (A.DICT_4X4_50, A.DICT_5X5_1000)), [(mc.grid(), 0), (mc.grid(), 1)], [], None),
    "absent_family": (GRIDS + [A.DICT_6X6_250], mc.render_grids, [(mc.grid(), 2), (mc.grid(), 0)], [(mc.charuco(), 2)], 2),
}


def _handle(dicts, method, inverted=False, enc="bgr8", max_batch=2):
    d = Detector(default_params(cornerRefinementMethod=method, dictionary=dicts[0]), max_width=W, max_height=H, max_batch=max_batch)
    if len(dicts) > 1:
        d.set_dictionaries(_specs(dicts))
    if inverted:
        d.set_detect_inverted_marker(True)
    if enc != "bgr8":
        d.set_input_encoding(enc)
    return d


def _bind(det, boards, charucos, dia, families=True):
    if boards:
        det.set_boards([b for b, _ in boards], [k for _, k in boards] if families else None)
    if charucos:
        det.set_charuco_boards([b for b, _ in charucos], [k for _, k in charucos] if families else None)
    if dia is not None:
        det.set_diamonds(mc.DIA_SQUARE, mc.DIA_MARKER, family=dia if families else None)


def _input(frames, enc):
    return np.ascontiguousarray(np.stack(frames)[..., 0] if enc == "mono8" else np.stack(frames))


def _run(det, frames, enc, cam, mode):
    x = _input(frames, enc)
    args = (K, D, 0.14) if cam else ()
    if mode == "batch":
        counts, ids, corners, _ = det.detect_pose_batch(x, *args)
    else:
        det.submit_batch(x, *args)
        counts, ids, corners, _ = det.collect_batch()
    return counts.copy(), ids.copy(), corners.copy().reshape(len(frames), MAXM, 4, 2), det.last_dict_indices()


_BOARD_FIELDS = ("status", "n_markers", "n_points", "rvec", "tvec", "rotation", "image_error")
_CH_FIELDS = ("status", "n_corners", "rvec", "tvec", "rotation", "image_error")


def _fields(r, names):
    return tuple(tuple(getattr(r, n)) if hasattr(getattr(r, n), "__len__") else getattr(r, n) for n in names)


def _check_frame(case, f, bgr, dicts, boards, charucos, dia, method, inverted, enc, cam, counts, ids, corners, di, brecs, chrecs, drecs):
    n = int(counts[f])
    ids, corners, di = ids[f, :n], corners[f, :n], di[f, :n]
    rids, _, rdi = mc.cv2_multi(bgr, dicts, method, inverted)
    assert ids.tolist() == rids.tolist() and di.tolist() == rdi.tolist(), (case, f)
    gray = np.ascontiguousarray(bgr[..., 0])  # the frames are gray
    frame = gray if enc == "mono8" else bgr
    for k, dk in enumerate(dicts):  # the single-dictionary handle of family k, fed corners[di == k]
        fi, fc = mc.family(ids, corners, di, k)
        mine_b = [j for j, (_, fam) in enumerate(boards) if fam == k]
        mine_c = [j for j, (_, fam) in enumerate(charucos) if fam == k]
        if not mine_b and not mine_c and dia != k:
            continue
        one = _handle([dk], method, inverted, enc, 1)
        _bind(one, [boards[j] for j in mine_b], [charucos[j] for j in mine_c], 0 if dia == k else None, families=False)
        if mine_b and cam:
            ref = one.board_poses(fi, fc, K, D)
            for i, j in enumerate(mine_b):
                assert _fields(brecs[f][j], _BOARD_FIELDS) == _fields(ref[i], _BOARD_FIELDS), (case, f, j)
                assert brecs[f][j].board == j
                bo.assert_matches(bo.record_dict(brecs[f][j]), bo.board_pose(boards[j][0], fi, fc, K, D), (case, f, j))
        if mine_c:
            ref = one.charuco(frame, fi, fc, K if cam else None, D if cam else None)
            for i, j in enumerate(mine_c):
                got, want = chrecs[f][j], ref[i]
                assert _fields(got[0], _CH_FIELDS) == _fields(want[0], _CH_FIELDS), (case, f, j)
                assert np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2]), (case, f, j)
                rid, rxy, rpose = co.full(mc.cv_charuco(charucos[j][0], dk), gray, fi, fc, K if cam else None, D if cam else None)
                gpose = dict(status=got[0].status, rvec=list(got[0].rvec), tvec=list(got[0].tvec), rotation=list(got[0].rotation), image_error=got[0].image_error)
                if not cam:
                    rpose = dict(rpose, status=0)
                co.assert_matches(got[1], got[2], gpose, rid, rxy, rpose, (case, f, j))
        if dia == k:
            sids, scorners, srecs = one.diamonds(frame, fi, fc, K if cam else None, D if cam else None)
            gids, gcorners, grecs = drecs[f]
            assert np.array_equal(gids, sids) and np.array_equal(gcorners, scorners), (case, f)
            for g, s in zip(grecs, srecs):
                assert g.pose.fiducial_id == s.pose.fiducial_id + OFFSETS[k] == g.ids[0] + OFFSETS[k]
                s.pose.fiducial_id = g.pose.fiducial_id
                assert bytes(g) == bytes(s), (case, f)
            if inverted:  # (the single-dictionary handle above pins this case)
                continue
            cids, ccorners = dio.detect(mc.diamond_detector(dk, K if cam else None, D if cam else None, method), gray, fi, fc)
            assert gids.tolist() == cids.tolist(), (case, f)
            if len(cids):
                assert np.abs(gcorners - ccorners).max() <= co.CORNER_TOL, (case, f)
            for g in grecs:
                if cam:
                    p = dio.pose(np.array(list(g.corners), np.float32).reshape(4, 2), mc.DIA_SQUARE, K, D)
                    assert np.abs(np.array(list(g.pose.translation)) - p["tvec"]).max() <= 1e-6, (case, f)
        one.close()


@pytest.mark.parametrize("case,method,cam,inverted,enc,mode", [
    ("grids_2", 1, True, False, "bgr8", "batch"),
    ("grids_2", 0, False, False, "mono8", "submit"),
    ("mixed_3", 1, True, False, "bgr8", "batch"),
    ("mixed_3", 0, False, False, "mono8", "submit"),
    ("mixed_3", 1, True, True, "mono8", "batch"),
    ("mixed_3_diamonds_in_36h11", 1, True, False, "bgr8", "submit"),
    ("listed_twice", 1, True, False, "bgr8", "batch"),
    ("absent_family", 1, True, False, "bgr8", "batch"),
])
def test_family_boards_match_cv2_and_single_dictionary_calls(case, method, cam, inverted, enc, mode):
    dicts, render, boards, charucos, dia = CASES[case]
    frames = [render(s) for s in (3, 4)]
    det = _handle(dicts, method, inverted, enc)
    _bind(det, boards, charucos, dia)
    counts, ids, corners, di = _run(det, frames, enc, cam, mode)
    brecs = det.last_board_poses() if boards and cam else None
    chrecs = det.last_charuco() if charucos else None
    drecs = det.last_diamonds() if dia is not None else None
    for f, bgr in enumerate(frames):
        _check_frame(case, f, bgr, dicts, boards, charucos, dia, method, inverted, enc, cam, counts, ids, corners, di, brecs, chrecs, drecs)
    if case == "absent_family":
        assert all(r[0].status == 0 for r in brecs) and all(c[0][0].n_corners == 0 for c in chrecs) and all(len(d[0]) == 0 for d in drecs)
    if case == "listed_twice" and cam:
        for r in brecs:
            assert _fields(r[0], _BOARD_FIELDS) == _fields(r[1], _BOARD_FIELDS) and r[0].status == 1
    if case.startswith("mixed") and dia is not None:
        assert sum(len(d[0]) for d in drecs) >= len(frames)


def _all_outputs(det, frames):
    counts, ids, corners, tfs = det.detect_pose_batch(np.stack(frames), K, D, 0.14)
    out = counts.tobytes() + ids.tobytes() + corners.tobytes() + bytes(tfs)
    out += b"".join(bytes(r) for fr in det.last_board_poses() for r in fr)
    out += b"".join(bytes(r[0]) + r[1].tobytes() + r[2].tobytes() for fr in det.last_charuco() for r in fr)
    out += b"".join(bytes(r) for fr in det.last_diamonds() for r in fr[2])
    return out


def test_index_zero_on_a_single_dictionary_handle_is_byte_identical():
    frames = [mc.render_mixed_boards(s) for s in (5, 6)]
    outs = []
    for fam in (False, True):
        det = _handle([A.DICT_6X6_250], 1)
        _bind(det, [(mc.grid(mc.DIA_IDS), 0)], [(mc.charuco(), 0)], 0, families=fam)
        outs.append(_all_outputs(det, frames))
        if fam:
            ids, corners = det.detect(frames[0])
            assert len(det.board_poses(ids, corners, K, D)) == 1  # the stand-alone calls work on a single-dictionary handle
    assert outs[0] == outs[1]


def test_validation_leaves_the_handle_unchanged():
    frames = [mc.render_mixed_boards(s) for s in (7, 8)]
    det = _handle(MIXED, 1)
    _bind(det, [(mc.grid(), 2)], [(mc.charuco(), 0)], 0)
    before = _all_outputs(det, frames)
    lib = det.lib
    arr = (_lib.fid_board * 1)()
    g = mc.grid()
    arr[0].n_markers, arr[0].ids, arr[0].obj_points = 4, g.ids.ctypes.data, g.obj_points.ctypes.data
    for bad in (3, -1):
        fam = np.array([bad], np.int32)
        assert lib.fid_set_family_boards(det.h, 1, C.cast(arr, C.c_void_p), fam.ctypes.data_as(C.c_void_p)) == -1
        with pytest.raises(_lib.FidError):
            det.set_charuco_boards([mc.charuco()], [bad])
        p = _lib.fid_diamond_params(1, mc.DIA_SQUARE, mc.DIA_MARKER, 2, 1)
        assert lib.fid_set_family_diamonds(det.h, C.byref(p), bad) == -1
    assert lib.fid_set_family_boards(det.h, 1, C.cast(arr, C.c_void_p), None) == -1
    # a list shrunk under a bound index, and a ChArUco board too large for its new family
    specs = lambda dl: (_lib.fid_dictionary_spec * len(dl))(*[_lib.fid_dictionary_spec(d, 0, 0.0) for d in dl])  # noqa: E731
    assert lib.fid_set_dictionaries(det.h, 2, C.cast(specs(MIXED[:2]), C.c_void_p)) == -1
    assert _all_outputs(det, frames) == before


def test_shrinking_to_a_dictionary_too_small_for_a_bound_charuco_board():
    from fiducials_b200.board import CharucoBoard

    det = _handle([A.DICT_5X5_1000, A.DICT_6X6_250], 1)
    det.set_charuco_boards([CharucoBoard((12, 10), 0.02, 0.015)], [0])  # 60 markers
    specs = (_lib.fid_dictionary_spec * 2)(_lib.fid_dictionary_spec(A.DICT_4X4_50, 0, 0.0), _lib.fid_dictionary_spec(A.DICT_6X6_250, 0, 0.0))
    assert det.lib.fid_set_dictionaries(det.h, 2, C.cast(specs, C.c_void_p)) == -1  # DICT_4X4_50 holds 50
    specs[0].dictionary = A.DICT_4X4_100
    assert det.lib.fid_set_dictionaries(det.h, 2, C.cast(specs, C.c_void_p)) == 0


def test_refusals_kept():
    frames = [mc.render_grids(9)]
    det = _handle(GRIDS, 1)
    for call in (lambda: det.set_boards([mc.grid()]), lambda: det.set_charuco_boards([mc.charuco()]), lambda: det.set_diamonds(0.04, 0.02)):
        with pytest.raises(_lib.FidError) as e:
            call()
        assert e.value.status == -4
    _bind(det, [(mc.grid(), 1)], [(mc.charuco(), 0)], 0)
    det.set_marker_refinement(10.0, 3.0, True)
    assert det.lib.fid_set_batch_marker_refinement(det.h, 1) == -4
    assert det.lib.fid_set_marker_confidence(det.h, 1) == -4
    ids, corners, _ = det.detect_multi_dict(frames[0])
    for call in (lambda: det.board_poses(ids, corners, K, D), lambda: det.charuco(frames[0], ids, corners), lambda: det.diamonds(frames[0], ids, corners),
                 lambda: det.refine_markers(frames[0], ids, corners, np.zeros((0, 4, 2), np.float32))):
        with pytest.raises(_lib.FidError) as e:
            call()
        assert e.value.status == -4


def test_node_per_frame_equals_batch():
    specs = [(A.DICT_6X6_250, 1000, 0.0), (A.DICT_APRILTAG_36h11, 2000, 0.0)]
    node = FiducialsNode(dictionary=A.DICT_4X4_50, fiducial_len=0.14, max_width=W, max_height=H, max_batch=2, dictionaries=specs,
                         boards=[(mc.grid(), 0), (mc.tags(), 2)], charuco_boards=[(mc.charuco(), 1)], diamonds=(mc.DIA_SQUARE, mc.DIA_MARKER, 1))
    node.camInfoCallback(K.reshape(-1), D, "camera")
    frames = [mc.render_mixed_boards(s) for s in (10, 11)]
    per = []
    for bgr in frames:
        per.append(node.poseEstimateCallback(node.imageCallback(bgr)))
    batch = node.process_batch(np.stack(frames))
    for p, b in zip(per, batch):
        assert [t.fiducial_id for t in p.transforms] == [t.fiducial_id for t in b.transforms]
        assert [bytes(r) for r in p.board_poses] == [bytes(r) for r in b.board_poses]
        assert all(r.status == 1 for r in p.board_poses)
        assert [bytes(r[0]) + r[1].tobytes() + r[2].tobytes() for r in p.charuco] == [bytes(r[0]) + r[1].tobytes() + r[2].tobytes() for r in b.charuco]
        assert [bytes(r) for r in p.diamonds[2]] == [bytes(r) for r in b.diamonds[2]]
        assert len(p.diamonds[2]) >= 1 and all(r.pose.fiducial_id == r.ids[0] + 1000 for r in p.diamonds[2])
        assert mc.DIA_IDS[0] in [r.ids[0] for r in p.diamonds[2]]
