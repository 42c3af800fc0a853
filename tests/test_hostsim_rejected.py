"""detectMarkers' rejectedImgPoints: the candidate hierarchy (fiducials_b200/csrc/candidate_tree.cuh, compiled for the host from
tests/hostsim/rejected_hostsim.cpp) on the host candidate stage, against cv2 4.13.  Count, order and corners must be identical.
CPU only."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import aruco_oracle as ao
import hostsim_util as hs
import rejected_cases as rc

_HERE = os.path.dirname(os.path.abspath(__file__))
_harness = None


def _load():
    """g++ build of the harness into a temporary directory (the tree may be read-only), once per session."""
    global _harness
    if _harness is None:
        tmp = tempfile.mkdtemp(prefix="fid_rejected_hostsim_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "libfid_rejected_hostsim.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, os.path.join(_HERE, "hostsim", "rejected_hostsim.cpp")])
        _harness = C.CDLL(so)
    return _harness


def hs_rejected(bgr, dict_id):
    """The host chain: ids in output order and the rejected list [m, 4, 2]."""
    g = ao.gray(bgr)
    quads, _, _ = hs.candidates(ao.threshold_planes(g), dict_id)
    H, W = g.shape
    raw = np.ascontiguousarray(quads.reshape(-1, 8), np.int32)
    ids = np.zeros(512, np.int32)
    rej = np.zeros((512, 8), np.float32)
    ni = C.c_int(0)
    vp = C.c_void_p
    n = _load().hs_rejected(np.ascontiguousarray(g).ctypes.data_as(vp), W, H, dict_id, len(raw), raw.ctypes.data_as(vp), ids.ctypes.data_as(vp), len(ids),
                            C.byref(ni), rej.ctypes.data_as(vp), len(rej))
    assert n >= 0, n
    return ids[: ni.value].copy(), rej[:n].reshape(-1, 4, 2).copy()


_seen = {"frames": 0, "rejected": 0}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nrejected lists vs cv2: %d frames, %d rejected candidates" % (_seen["frames"], _seen["rejected"]))


def check(name, bgr, dict_id):
    ids, rej = hs_rejected(bgr, dict_id)
    rids, _, rrej = rc.cv2_lists(bgr, dict_id)
    assert ids.tolist() == rids.tolist(), name
    assert len(rej) == len(rrej), (name, len(rej), len(rrej))
    assert np.array_equal(rej, rrej), (name, rej, rrej)  # same order, bit-identical corners
    _seen["frames"] += 1
    _seen["rejected"] += len(rej)
    return len(rej)


@pytest.mark.parametrize("case", list(range(7)))
def test_synthetic_frames(case):
    name, bgr, d = list(rc.synthetic_frames())[case]
    n = check(name, bgr, d)
    if name == "C2/0":
        assert n == 7  # what cv2 returns there


def test_reference_frames(kat):
    for name in ("tag01", "tag245", "img403", "bag"):
        check(name, kat.frame(name), 7)


def test_border_frames():
    for name, bgr, d in rc.border_frames():
        check(name, bgr, d)


def test_nested_markers():
    """The enclosing marker is rejected when its level is never reached (first frame) and a marker when it is (second)."""
    sizes = [check(name, bgr, d) for name, bgr, d in rc.nested_frames()]
    assert len(sizes) == 2


def test_damaged_boards():
    total = sum(check(name, bgr, d) for name, bgr, d in rc.damaged_frames())
    assert total > 0
