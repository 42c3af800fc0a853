"""The dense calibration-target cases of tests/dense_cases.py stay in the size bands they were chosen for: raw quad candidates under the
oracle, selected candidates and markers under the host build of the device's grouping and identification, markers under cv2.
A change to the generator that moves a case out of its band fails here, on the CPU, before the GPU tests lose the path it covers.
CPU only."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

import dense_cases as dc
from oracle import aruco_oracle as ao

FID_MAX_RAW, FID_MAX_SEL, FID_MAX_MARKERS = 4096, 512, 256
_HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def harness():
    """g++ build of tests/dense_hostsim.cpp into a temporary directory (the tree may be read-only)."""
    tmp = tempfile.mkdtemp(prefix="fid_dense_hostsim_")
    atexit.register(shutil.rmtree, tmp, True)
    so = os.path.join(tmp, "libfid_dense_hostsim.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, os.path.join(_HERE, "dense_hostsim.cpp")])
    lib = C.CDLL(so)
    lib.hs_dense_counts.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, C.c_void_p, C.c_int, C.c_void_p]
    return lib


def host_counts(lib, g, planes, dict_id, p):
    """The host chain's markers (ids in OpenCV's order), raw and selected candidate counts."""
    g = np.ascontiguousarray(g, np.uint8)
    planes = np.ascontiguousarray(planes, np.uint8)
    H, W = g.shape
    ids = np.zeros(1024, np.int32)
    stats = np.zeros(2, np.int32)
    n = lib.hs_dense_counts(g.ctypes.data, planes.ctypes.data, W, H, dict_id, p["adaptiveThreshWinSizeMin"], p["adaptiveThreshWinSizeMax"],
                            p["adaptiveThreshWinSizeStep"], p["minMarkerPerimeterRate"], ids.ctypes.data, len(ids), stats.ctypes.data)
    assert n >= 0, n
    return ids[:n].copy(), int(stats[0]), int(stats[1])


@pytest.mark.parametrize("name", sorted(dc.CASES))
def test_case_stays_in_its_band(harness, name):
    c = dc.CASES[name]
    bgr, rendered = dc.render(name)
    assert bgr.shape == (c["H"], c["W"], 3)
    p = dc.oracle_params(name)
    g = ao.gray(bgr)
    raw = len(ao.quad_candidates(g, p))
    lo, hi = dc.BANDS[c["band"]]
    assert lo <= raw <= hi, (name, raw, c["band"])
    kw = dict(c["params"], detectInvertedMarker=True) if c["inverted"] else c["params"]
    rids, _ = ao.detect(bgr, c["dict_id"], **kw)
    assert len(rids) == dc.MARKERS[name] and len(set(rids.tolist())) == len(rids) and set(rids.tolist()) <= rendered
    if c["inverted"]:
        return  # the host harness reads black-on-white markers only; the candidate stage above is the same for both polarities
    ids, host_raw, sel = host_counts(harness, g, ao.threshold_planes(g, p), c["dict_id"], p)
    assert host_raw == raw  # the host build of the candidate stage finds the oracle's candidates
    assert ids.tolist() == rids.tolist()
    assert (sel > FID_MAX_SEL) == (name == "grid_32x18_few"), (name, sel)
    assert sel >= len(ids)


def test_cases_cross_every_capacity():
    """Together the cases cross n = 615, 1537, 2049 and 4096 raw candidates, 256 markers and 512 selected, and the bands each have a
    case (the sizes at which k_sort_group and k_finish switch paths, dense_cases.py)."""
    bands = {c["band"] for c in dc.CASES.values()}
    assert bands == set(dc.BANDS)
    m = dc.MARKERS
    assert any(v == FID_MAX_MARKERS for v in m.values()) and any(v > FID_MAX_MARKERS for k, v in m.items() if dc.CASES[k]["band"] != "gt4096")
    assert any(v <= FID_MAX_MARKERS for k, v in m.items() if dc.CASES[k]["band"] == "gt4096")
