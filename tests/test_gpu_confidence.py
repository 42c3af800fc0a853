"""Detection with confidence on the device (fid_detect_with_confidence, fid_set_marker_confidence, fid_last_marker_confidence): bit for
bit against the host chain (tests/hostsim/confidence_hostsim.cpp) and against cv2's detectMarkersWithConfidence; the batch calls
with the option on equal the single-frame call and leave ids, corners and transforms byte-identical; the refusals."""
import ctypes as C

import cv2
import numpy as np
import pytest

from fiducials_b200 import _lib
from fiducials_b200.node import MAXM, Detector
import confidence_oracle as co

pytestmark = pytest.mark.gpu
A = co.A
FID_ERR_INVALID_ARG, FID_ERR_UNSUPPORTED, FID_ERR_CAPACITY = -1, -4, -5
K = np.array([[600.0, 0, 320], [0, 600.0, 240], [0, 0, 1]])
D = np.zeros(5)


def _bgr(g):
    return np.ascontiguousarray(cv2.cvtColor(g, cv2.COLOR_GRAY2BGR))


def _det(dict_id, max_batch=4, **kw):
    return Detector(co.fid_params_for(dict_id, **kw), max_width=640, max_height=480, max_batch=max_batch)


def _tf_bytes(tfs, counts, n_frames):
    raw = bytes(tfs)
    rec = C.sizeof(_lib.fid_transform)
    return [raw[f * MAXM * rec:(f * MAXM + int(counts[f])) * rec] for f in range(n_frames)]


@pytest.mark.parametrize("case", list(co.sweep_cases(60)), ids=lambda c: c[0])
def test_single_frame_matches_host_and_cv2(case):
    name, g, dict_id, kw = case
    det = _det(dict_id, max_batch=1, **kw)
    ids, corners, conf = det.detect_with_confidence(_bgr(g))
    hi, hc, hf = co.host_detect(g, dict_id, **kw)
    assert ids.tolist() == hi.tolist()
    assert np.array_equal(corners, hc)
    assert np.array_equal(conf.view(np.int32), hf.view(np.int32))
    pi, pc = det.detect(_bgr(g))  # ids and corners exactly as fid_detect
    assert np.array_equal(pi, ids) and np.array_equal(pc, corners)
    ci, _, cf = co.cv2_detect(g, dict_id, **kw)
    assert ci.tolist() == ids.tolist()
    assert np.abs(cf.astype(np.float64) - conf).max(initial=0) <= 1e-6


@pytest.mark.parametrize("case", co.fixed_cases(), ids=lambda c: c[0])
def test_fixed_cases(case):
    name, g, dict_id, kw, expected = case
    ids, _, conf = _det(dict_id, max_batch=1, **kw).detect_with_confidence(_bgr(g))
    assert len(ids) == 1 and conf[0] == np.float32(expected)


@pytest.mark.parametrize("method", ["none", "subpix", "contour"])
def test_batch_equals_single_frame_and_leaves_outputs_unchanged(method):
    cases = [c for c in co.sweep_cases(60) if c[2] == A.DICT_6X6_250][:6]
    frames = np.ascontiguousarray(np.stack([_bgr(c[1]) for c in cases]))
    kw = dict(method=method, border_bits=1, ppc=8, margin=0.13)
    det = _det(A.DICT_6X6_250, **kw)
    off = [np.copy(x) for x in det.detect_pose_batch(frames, K, D, 0.14)[:3]]
    off_tf = _tf_bytes(det.detect_pose_batch(frames, K, D, 0.14)[3], off[0], len(frames))
    with pytest.raises(_lib.FidError) as e:
        det.last_marker_confidence()
    assert e.value.status == FID_ERR_INVALID_ARG
    det.set_marker_confidence(True)
    counts, ids, corners, tfs = det.detect_pose_batch(frames, K, D, 0.14)
    assert np.array_equal(counts, off[0]) and np.array_equal(ids, off[1]) and np.array_equal(corners, off[2])
    assert _tf_bytes(tfs, counts, len(frames)) == off_tf
    conf = det.last_marker_confidence()
    assert conf.shape == (len(frames), MAXM) and int(counts.sum()) > 10
    single = _det(A.DICT_6X6_250, max_batch=1, **kw)
    for f, fr in enumerate(frames):
        si, sc, sf = single.detect_with_confidence(fr)
        n = int(counts[f])
        assert si.tolist() == ids[f, :n].tolist()
        assert np.array_equal(sf.view(np.int32), conf[f, :n].view(np.int32))
    # capacity: nothing written when a frame has more markers than max_markers
    small = np.full((len(frames), 1), -7.0, np.float32)
    nf = C.c_int(0)
    st = det.lib.fid_last_marker_confidence(det.h, 1, C.byref(nf), small.ctypes.data_as(C.c_void_p))
    assert st == FID_ERR_CAPACITY and (small == -7.0).all() and nf.value == len(frames)
    # off again: the batch outputs are restored and the confidence is refused
    det.set_marker_confidence(False)
    c2, i2, k2, _ = det.detect_pose_batch(frames, K, D, 0.14)
    assert np.array_equal(c2, off[0]) and np.array_equal(i2, off[1]) and np.array_equal(k2, off[2])
    with pytest.raises(_lib.FidError):
        det.last_marker_confidence()


@pytest.mark.parametrize("encoding", ["bgr8", "rgb8", "mono8"])
def test_submit_collect_two_batches_in_flight(encoding):
    cases = [c for c in co.sweep_cases(90) if c[2] == A.DICT_APRILTAG_36h11][:6]
    grays = [c[1] for c in cases]
    if encoding == "mono8":
        frames = np.ascontiguousarray(np.stack(grays))
    elif encoding == "rgb8":
        frames = np.ascontiguousarray(np.stack([cv2.cvtColor(g, cv2.COLOR_GRAY2RGB) for g in grays]))
    else:
        frames = np.ascontiguousarray(np.stack([_bgr(g) for g in grays]))
    det = _det(A.DICT_APRILTAG_36h11, max_batch=3)
    det.set_input_encoding(encoding)
    det.set_marker_confidence(True)
    det.submit_batch(frames[:3], K, D, 0.14)
    det.submit_batch(frames[3:], K, D, 0.14)
    with pytest.raises(_lib.FidError):  # not while batches are in flight
        det.set_marker_confidence(False)
    for b in range(2):
        counts, ids, _, _ = det.collect_batch()
        conf = det.last_marker_confidence()
        for f in range(3):
            g = grays[3 * b + f]
            hi, _, hf = co.host_detect(g, A.DICT_APRILTAG_36h11)
            n = int(counts[f])
            assert ids[f, :n].tolist() == hi.tolist()
            assert np.array_equal(conf[f, :n].view(np.int32), hf.view(np.int32))


def test_aruco3_matches_cv2():
    """With useAruco3Detection the confidence comes from the pyramid level the bits are read from."""
    n = 0
    for name, g, dict_id, kw in list(co.sweep_cases(40))[:20]:
        det = _det(dict_id, max_batch=1, **kw)
        det.set_aruco3(32, 0.02)
        ids, _, conf = det.detect_with_confidence(_bgr(g))
        ci, _, cf = co.cv2_detect(g, dict_id, aruco3=(32, 0.02), **kw)
        assert ids.tolist() == ci.tolist(), name
        assert np.abs(cf.astype(np.float64) - conf).max(initial=0) <= 1e-6, name
        n += len(ids)
    assert n > 20


def test_refusals():
    det = _det(A.DICT_6X6_250)
    det.set_dictionaries([A.DICT_6X6_250, A.DICT_4X4_50])
    for call in (lambda: det.set_marker_confidence(True), lambda: det.detect_with_confidence(np.zeros((480, 640, 3), np.uint8))):
        with pytest.raises(_lib.FidError) as e:
            call()
        assert e.value.status == FID_ERR_UNSUPPORTED
    det = _det(A.DICT_6X6_250)
    det.set_marker_confidence(True)
    with pytest.raises(_lib.FidError) as e:
        det.set_dictionaries([A.DICT_6X6_250, A.DICT_4X4_50])
    assert e.value.status == FID_ERR_UNSUPPORTED
    det.set_marker_refinement()
    with pytest.raises(_lib.FidError) as e:
        det.set_batch_marker_refinement(True)
    assert e.value.status == FID_ERR_UNSUPPORTED
    det.set_marker_confidence(False)
    det.set_batch_marker_refinement(True)
    with pytest.raises(_lib.FidError) as e:
        det.set_marker_confidence(True)
    assert e.value.status == FID_ERR_UNSUPPORTED
