"""White-on-black markers on the device (fid_set_detect_inverted_marker, cv2's detectInvertedMarker): bit for bit against the host
chain (tests/hostsim/inverted_hostsim.cpp) and against cv2 4.13, for single frames, batches and submit/collect in every encoding and
with both threshold kernels; the flag set and cleared leaves a handle as it was; poses, boards, ChArUco and diamonds read the final
markers; several dictionaries, useAruco3Detection and confidence; the refusals; the node and its C++ glue."""
import ctypes as C
import os
import subprocess

import cv2
import numpy as np
import pytest

from fiducials_b200 import _lib, synth
from fiducials_b200.node import MAXM, Detector, FiducialsNode, default_params
import inverted_oracle as io

pytestmark = pytest.mark.gpu
A = io.A
FID_ERR_INVALID_ARG, FID_ERR_UNSUPPORTED = -1, -4
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = {"none": 0.0, "subpix": 0.05, "contour": 0.05}  # corners against cv2 (tests/test_hostsim_inverted.py has the derivation)


def _bgr(g):
    return np.ascontiguousarray(cv2.cvtColor(g, cv2.COLOR_GRAY2BGR))


def _det(dict_id, W=640, H=480, max_batch=1, inverted=True, **kw):
    det = Detector(io.fid_params_for(dict_id, **kw), max_width=W, max_height=H, max_batch=max_batch)
    if inverted:
        det.set_detect_inverted_marker(True)
    return det


def _tf_bytes(tfs, counts, n_frames):
    raw = bytes(tfs)
    rec = C.sizeof(_lib.fid_transform)
    return [raw[f * MAXM * rec:(f * MAXM + int(counts[f])) * rec] for f in range(n_frames)]


@pytest.mark.parametrize("case", list(io.sweep_cases(60)), ids=lambda c: c[0])
def test_single_frame_matches_host_and_cv2(case):
    name, g, dict_id, kw = case
    H, W = g.shape
    det = _det(dict_id, W, H, **kw)
    ids, corners = det.detect(_bgr(g))
    hi, hc, hf, _ = io.host_detect(g, dict_id, **kw)
    assert ids.tolist() == hi.tolist()
    assert np.array_equal(corners, hc)
    ci, cc, _ = io.cv2_detect(g, dict_id, **kw)
    assert ci.tolist() == ids.tolist()
    assert np.abs(cc - corners).max(initial=0) <= TOL[kw["method"]]
    qi, qc, qf = det.detect_with_confidence(_bgr(g))
    assert np.array_equal(qi, ids) and np.array_equal(qc, corners)
    assert np.array_equal(qf.view(np.int32), hf.view(np.int32))


def test_blank_frames():
    det = _det(A.DICT_6X6_250)
    for name, g in io.blank_frames():
        ids, _ = det.detect(_bgr(g))
        assert ids.tolist() == io.host_detect(g, A.DICT_6X6_250)[0].tolist() == io.cv2_detect(g, A.DICT_6X6_250)[0].tolist(), name


def _frames(encoding, seed, n=6, dict_id=A.DICT_6X6_250):
    grays = [io.render(seed + i, dict_id, 1, "clean", io.POLARITIES[i % 3], n_markers=8) for i in range(n)]
    if encoding == "mono8":
        frames = np.stack(grays)
    elif encoding == "rgb8":
        frames = np.stack([cv2.cvtColor(g, cv2.COLOR_GRAY2RGB) for g in grays])
    else:
        frames = np.stack([_bgr(g) for g in grays])
    return grays, np.ascontiguousarray(frames)


@pytest.mark.parametrize("thresh", ["default", "mma"])
@pytest.mark.parametrize("encoding", ["bgr8", "rgb8", "mono8"])
def test_batches_and_submit_collect_match_host(monkeypatch, encoding, thresh):
    if thresh == "mma":
        monkeypatch.setenv("FID_THRESH", "mma")  # read by fid_create
    grays, frames = _frames(encoding, 300)
    det = _det(A.DICT_6X6_250, max_batch=3)
    det.set_input_encoding(encoding)
    counts, ids, corners, _ = det.detect_pose_batch(frames)
    counts, ids, corners = counts.copy(), ids.copy(), corners.copy()
    det.submit_batch(frames[:3])
    det.submit_batch(frames[3:])
    with pytest.raises(_lib.FidError) as e:  # not while batches are in flight
        det.set_detect_inverted_marker(False)
    assert e.value.status == FID_ERR_INVALID_ARG
    collected = [det.collect_batch() for _ in range(2)]
    n_white = 0
    for f, g in enumerate(grays):
        hi, hc, _, hp = io.host_detect(g, A.DICT_6X6_250)
        n = int(counts[f])
        assert ids[f, :n].tolist() == hi.tolist(), f
        assert np.array_equal(corners[f, :n], hc), f
        cc, ci, ck, _ = collected[f // 3]
        assert int(cc[f % 3]) == n and ci[f % 3, :n].tolist() == hi.tolist() and np.array_equal(ck[f % 3, :n], hc)
        n_white += int(hp.sum())
    assert n_white >= 10 and int(counts.sum()) >= 30


def test_set_and_clear_leaves_handle_as_untouched():
    """With the flag set and cleared again, every output is byte-identical with a handle that was never touched; with it on, the
    transforms are those of fid_pose on the same corners."""
    grays, frames = _frames("bgr8", 400)
    K, D = synth.camera_for(640, 480)
    plain = _det(A.DICT_6X6_250, max_batch=6, inverted=False)
    ref = plain.detect_pose_batch(frames, K, D, 0.14)
    ref = (ref[0].copy(), ref[1].copy(), ref[2].copy(), _tf_bytes(ref[3], ref[0], len(frames)))
    det = _det(A.DICT_6X6_250, max_batch=6)
    on = det.detect_pose_batch(frames, K, D, 0.14)
    assert not np.array_equal(on[2], ref[2])  # the flag changes black markers' corners (DESIGN.md finding 18 B)
    for f in range(len(frames)):
        n = int(on[0][f])
        tfs = det.pose(on[1][f, :n], on[2][f, :n], K, D, 0.14)
        assert b"".join(bytes(t) for t in tfs) == _tf_bytes(on[3], on[0], len(frames))[f]
    det.set_detect_inverted_marker(False)
    off = det.detect_pose_batch(frames, K, D, 0.14)
    assert np.array_equal(off[0], ref[0])
    for f in range(len(frames)):  # entries past counts[f] are not written
        n = int(off[0][f])
        assert np.array_equal(off[1][f, :n], ref[1][f, :n]) and np.array_equal(off[2][f, :n], ref[2][f, :n])
    assert _tf_bytes(off[3], off[0], len(frames)) == ref[3]
    for g in grays[:2]:
        a, b = plain.detect(_bgr(g)), det.detect(_bgr(g))
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def _cv2_multi(g, dict_ids):
    p = io.cv2_params(True)
    det = A.ArucoDetector(A.getPredefinedDictionary(dict_ids[0]), p)
    det.setDictionaries([A.getPredefinedDictionary(d) for d in dict_ids])
    corners, ids, _, di = det.detectMarkersMultiDict(g)
    if ids is None or len(ids) == 0:
        return np.zeros(0, np.int32), np.zeros((0, 4, 2), np.float32), np.zeros(0, np.int32)
    return ids.reshape(-1).astype(np.int32), np.array(corners, np.float32).reshape(-1, 4, 2), np.asarray(di).reshape(-1).astype(np.int32)


def test_multi_dict_matches_cv2():
    dicts = [A.DICT_6X6_250, A.DICT_4X4_50]
    n = n_off = 0
    for s in range(4):
        g = np.concatenate([io.render(500 + s, dicts[0], polarity="mixed"), io.render(600 + s, dicts[1], polarity=("inverted", "mixed")[s % 2])], axis=1)
        g = np.ascontiguousarray(g)
        H, W = g.shape
        det = _det(dicts[0], W, H)
        det.set_dictionaries(dicts)
        ids, corners, di = det.detect_multi_dict(_bgr(g))
        ci, cc, cdi = _cv2_multi(g, dicts)
        assert ids.tolist() == ci.tolist() and di.tolist() == cdi.tolist(), s
        assert np.abs(cc - corners).max(initial=0) <= TOL["subpix"]
        n += len(ids)
        det.set_detect_inverted_marker(False)
        n_off += len(det.detect_multi_dict(_bgr(g))[0])
    assert n > n_off + 8, (n, n_off)


def test_aruco3_matches_cv2():
    n = 0
    for name, g, dict_id, kw in list(io.sweep_cases(30))[:15]:
        H, W = g.shape
        det = _det(dict_id, W, H, **kw)
        det.set_aruco3(32, 0.02)
        ids, corners = det.detect(_bgr(g))
        ci, cc, _ = io.cv2_detect(g, dict_id, aruco3=(32, 0.02), **kw)
        assert ids.tolist() == ci.tolist(), name
        assert np.abs(cc - corners).max(initial=0) <= 1e-3, name  # finding 16: a few corners differ in the last bits
        n += len(ids)
    assert n > 30


def test_confidence_of_white_markers_matches_cv2():
    """4 pixels per cell, no margin: every share is a dyadic fraction, so cv2's confidences are matched exactly."""
    n = n_below = 0
    for s in range(6):
        g = io.render(800 + s, A.DICT_5X5_1000, 1, "noise", ("inverted", "mixed")[s % 2])
        det = _det(A.DICT_5X5_1000, ppc=4, margin=0.0)
        ids, _, conf = det.detect_with_confidence(_bgr(g))
        ci, _, cf = io.cv2_detect_conf(g, A.DICT_5X5_1000, ppc=4, margin=0.0)
        assert ids.tolist() == ci.tolist()
        assert np.array_equal(conf.view(np.int32), cf.view(np.int32))
        n += len(ids)
        n_below += int((conf < 1).sum())
    assert n > 20 and n_below > 5


def test_boards_charuco_and_diamonds_read_the_final_markers():
    """White boards (inverted frames): each batch record equals the stand-alone call on the batch's own markers."""
    import test_gpu_board_pose as tb
    import test_gpu_charuco as tc
    import test_gpu_diamond as td

    frames = np.ascontiguousarray(255 - tb.rendered_frames(8, seed=3)[0])
    det = Detector(default_params(dictionary=tb.DICT_ID), 0, tb.W, tb.H, 4)
    det.set_detect_inverted_marker(True)
    det.set_boards([tb.BOARD_A, tb.BOARD_B])
    counts, ids, corners, _ = det.detect_pose_batch(frames, tb.K_R, tb.D_ZERO, tb.FLEN)
    recs = det.last_board_poses()
    corners = corners.reshape(len(frames), MAXM, 8)
    for f in range(len(frames)):
        lst = det.board_poses(ids[f, :counts[f]], corners[f, :counts[f]], tb.K_R, tb.D_ZERO)
        assert [bytes(r) for r in lst] == [bytes(r) for r in recs[f]]
    assert sum(r.status == 1 for fr in recs for r in fr) >= 2
    det.close()

    frames = np.ascontiguousarray(255 - tc._frames(6, 4, [tc.BOARD_A, tc.BOARD_B]))
    det = Detector(default_params(dictionary=tc.co.DICT_ID), 0, tc.W, tc.H, 4)
    det.set_detect_inverted_marker(True)
    det.set_charuco_boards([tc.BOARD_A, tc.BOARD_B])
    det.submit_batch(frames, tc.K_R, tc.D_ZERO, tc.FLEN)
    counts, ids, corners, _ = det.collect_batch()
    ch = det.last_charuco()
    corners = corners.reshape(len(frames), MAXM, 8)
    n_corners = 0
    for f in range(len(frames)):
        n = int(counts[f])
        single = det.charuco(frames[f], ids[f, :n], corners[f, :n], tc.K_R, tc.D_ZERO)
        for (r1, i1, x1), (r2, i2, x2) in zip(ch[f], single):
            assert bytes(r1) == bytes(r2) and np.array_equal(i1, i2) and np.array_equal(x1, x2)
            n_corners += len(i1)
    assert n_corners > 0
    det.close()

    frames = np.ascontiguousarray(255 - td._frames(6, 5))
    det = Detector(default_params(dictionary=td.do.DICT_ID), 0, td.W, td.H, 4)
    det.set_detect_inverted_marker(True)
    det.set_diamonds(td.SQ, td.MK)
    counts, ids, corners, _ = det.detect_pose_batch(frames, td.K_SYN, td.D_ZERO, td.FLEN)
    dia = det.last_diamonds()
    corners = corners.reshape(len(frames), MAXM, 8)
    for f in range(len(frames)):
        n = int(counts[f])
        si, sc, srec = det.diamonds(frames[f], ids[f, :n], corners[f, :n], td.K_SYN, td.D_ZERO)
        bi, bc, brec = dia[f]
        assert np.array_equal(bi, si) and np.array_equal(bc, sc) and [bytes(r) for r in brec] == [bytes(r) for r in srec], f
    assert sum(len(d[0]) for d in dia) >= 1
    det.close()


def test_refusals():
    g = io.render(900, A.DICT_6X6_250, polarity="mixed")
    det = _det(A.DICT_6X6_250, max_batch=2)
    det.detect(_bgr(g))
    for call in (lambda: det.debug_rejected(), lambda: det.set_batch_marker_refinement(True), lambda: det.set_marker_refinement()):
        with pytest.raises(_lib.FidError) as e:
            call()
        assert e.value.status == FID_ERR_UNSUPPORTED
    # fid_refine_detected_markers: refused while the flag is on
    lib = det.lib
    bgr = _bgr(g)
    ids = np.zeros(4, np.int32)
    corners = np.zeros((4, 8), np.float32)
    idx, brd = np.zeros(4, np.int32), np.zeros(4, np.int32)
    n_out = C.c_int(0)
    st = lib.fid_refine_detected_markers(det.h, bgr.ctypes.data_as(C.c_void_p), 640, 480, 640 * 3, 0, ids.ctypes.data_as(C.c_void_p), corners.ctypes.data_as(C.c_void_p), 4,
                                         0, None, None, C.byref(n_out), idx.ctypes.data_as(C.c_void_p), brd.ctypes.data_as(C.c_void_p))
    assert st == FID_ERR_UNSUPPORTED
    # nothing changed: still on, still detecting white markers
    assert det.detect(_bgr(g))[0].tolist() == io.host_detect(g, A.DICT_6X6_250)[0].tolist()
    # the other direction
    det = _det(A.DICT_6X6_250, max_batch=2, inverted=False)
    det.set_marker_refinement()
    with pytest.raises(_lib.FidError) as e:
        det.set_detect_inverted_marker(True)
    assert e.value.status == FID_ERR_UNSUPPORTED
    det = _det(A.DICT_6X6_250, max_batch=2, inverted=False)
    det.set_marker_refinement()
    det.set_batch_marker_refinement(True)
    with pytest.raises(_lib.FidError) as e:
        det.set_detect_inverted_marker(True)
    assert e.value.status == FID_ERR_UNSUPPORTED
    # off again: the rejected list is available after the next detection
    det = _det(A.DICT_6X6_250)
    det.set_detect_inverted_marker(False)
    det.detect(_bgr(g))
    det.debug_rejected()


NW, NH = 1280, 720


def _node_frames(n, seed):
    return [_bgr(io.render(seed + i, A.DICT_6X6_250, 1, "clean", ("inverted", "mixed")[i % 2], NW, NH, n_markers=10)) for i in range(n)]


def _key(t):
    return (t.fiducial_id, t.transform.translation, t.transform.rotation, t.image_error, t.object_error, t.fiducial_area)


def test_node_per_frame_equals_batch():
    frames = _node_frames(3, 1000)
    K, D = synth.camera_for(NW, NH)
    per_frame = FiducialsNode(dictionary=A.DICT_6X6_250, fiducial_len=0.14, max_width=NW, max_height=NH, detect_inverted_marker=True)
    batch = FiducialsNode(dictionary=A.DICT_6X6_250, fiducial_len=0.14, max_width=NW, max_height=NH, max_batch=4, detect_inverted_marker=True)
    for node in (per_frame, batch):
        node.camInfoCallback(K, D, "camera")
    msgs = batch.process_batch(np.stack(frames))
    n = 0
    for f, bgr in enumerate(frames):
        fva = per_frame.imageCallback(bgr)
        fta = per_frame.poseEstimateCallback(fva)
        ids, corners, _, _ = io.host_detect(bgr, A.DICT_6X6_250)
        assert [v.fiducial_id for v in fva.fiducials] == ids.tolist()
        got_c = np.array([[v.x0, v.y0, v.x1, v.y1, v.x2, v.y2, v.x3, v.y3] for v in fva.fiducials], np.float32).reshape(-1, 4, 2)
        assert np.array_equal(got_c, corners)
        assert [_key(t) for t in fta.transforms] == [_key(t) for t in msgs[f].transforms]
        n += len(fta.transforms)
    assert n >= 15


def test_node_glue_matches_python_node(tmp_path):
    from test_node_glue import _build  # builds the library if needed

    _build()
    exe = str(tmp_path / "node_glue_inverted_main")
    libdir = os.path.join(ROOT, "fiducials_b200")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "node_glue_inverted_main.cpp"), "-L" + libdir, "-lfiducials_b200",
                           "-Wl,-rpath," + libdir, "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64", "-lcudart"])
    bgr = _node_frames(1, 1100)[0]
    raw = tmp_path / "f.bgr"
    raw.write_bytes(bgr.tobytes())
    r = subprocess.run([exe, str(raw), str(NW), str(NH), str(A.DICT_6X6_250), "0.14"], capture_output=True, text=True, check=True)
    node = FiducialsNode(dictionary=A.DICT_6X6_250, fiducial_len=0.14, max_width=NW, max_height=NH, detect_inverted_marker=True)
    K = np.array([[0.73 * NW, 0, NW / 2.0], [0, 0.73 * NW, NH / 2.0], [0, 0, 1]])
    node.camInfoCallback(K, [-0.2, 0.05, 0.001, -0.001, 0.0], "camera")
    fva = node.imageCallback(bgr)
    fta = node.poseEstimateCallback(fva)
    V = [l.split() for l in r.stdout.splitlines() if l.startswith("V ")]
    T = [l.split() for l in r.stdout.splitlines() if l.startswith("T ")]
    assert [int(v[1]) for v in V] == [v.fiducial_id for v in fva.fiducials] == io.host_detect(bgr, A.DICT_6X6_250)[0].tolist()
    got = np.array([[v.x0, v.y0, v.x1, v.y1, v.x2, v.y2, v.x3, v.y3] for v in fva.fiducials], np.float32)
    assert np.array_equal(np.array([[float(x) for x in v[2:]] for v in V], np.float32), got)
    assert len(T) == len(fta.transforms) > 3
    for t, m in zip(T, fta.transforms):
        assert int(t[1]) == m.fiducial_id
        vals = [float(x) for x in t[2:]]
        assert vals == list(m.transform.translation) + list(m.transform.rotation) + [m.image_error, m.object_error, m.fiducial_area]
