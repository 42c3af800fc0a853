"""Both planar pose hypotheses of a square marker (fiducials_b200/csrc/ippe.cuh, compiled for the host from
tests/hostsim/ippe_hostsim.cpp) against cv2.solvePnPGeneric(SOLVEPNP_IPPE_SQUARE).  CPU only."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import cv2
import numpy as np
import pytest

from fiducials_b200 import synth
import ippe_oracle as io

_HERE = os.path.dirname(os.path.abspath(__file__))
_harness = None


def _load():
    """g++ build of the harness into a temporary directory (the tree may be read-only), once per session; the flags of
    tests/hostsim/build.sh (no FMA contraction, like the device build)."""
    global _harness
    if _harness is None:
        tmp = tempfile.mkdtemp(prefix="fid_ippe_hostsim_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "libfid_ippe_hostsim.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, os.path.join(_HERE, "hostsim", "ippe_hostsim.cpp")])
        _harness = C.CDLL(so)
    return _harness


K_SYN, D_REF = synth.camera_for(640, 480)
D_ZERO = np.zeros(5)


def hs_hypotheses(corners, K, D, lens):
    """ippe.cuh on the host: list of dicts like ippe_oracle.pose_hypotheses."""
    lib = _load()
    c = np.ascontiguousarray(corners, np.float32).reshape(-1, 8)
    n = len(c)
    K = np.ascontiguousarray(K, np.float64).reshape(9)
    D = np.ascontiguousarray(D, np.float64).reshape(-1)[:5]
    lens = np.ascontiguousarray(lens, np.float32)
    out = np.zeros((n, 24))
    lib.hs_pose_hypotheses(n, c.ctypes.data_as(C.c_void_p), K.ctypes.data_as(C.c_void_p), D.ctypes.data_as(C.c_void_p), lens.ctypes.data_as(C.c_void_p),
                           out.ctypes.data_as(C.c_void_p))
    return [dict(n=int(o[0]), iterative_match=int(o[1]), rvec=o[2:8].reshape(2, 3), tvec=o[8:14].reshape(2, 3), rms=o[14:16], solver_err=o[16:18],
                 iterative_rvec=o[18:21]) for o in out]


def _check(cases, K, D):
    corners = np.array([c for c, _ in cases])
    lens = np.array([L for _, L in cases], np.float32)
    got = hs_hypotheses(corners, K, D, lens)
    n_close = 0
    for i, (c, L) in enumerate(cases):
        ref = io.pose_hypotheses(c, K, D, L)
        io.assert_matches(got[i], ref, "case %d" % i)
        if ref["n"] and ref["rms"][1] < 2.0 * ref["rms"][0]:
            n_close += 1
    return n_close


@pytest.mark.parametrize("name", ["tag01", "tag245", "img403", "bag"])
def test_golden_frames(kat, name):
    corners = kat[name + "_corners"]
    L = float(np.float32(float(kat[name + "_len"])))
    _check([(c, L) for c in corners], kat[name + "_K"].reshape(3, 3), kat[name + "_D"])


@pytest.mark.parametrize("D", [D_REF, D_ZERO], ids=["D_ref", "D_zero"])
@pytest.mark.parametrize("kind,seed", [("far", 1), ("far", 2), ("tilted", 3), ("mixed", 4)])
def test_synthetic(kind, seed, D):
    n_close = _check(io.synthetic_cases(seed, K_SYN, D, kind=kind), K_SYN, D)
    if kind == "far":  # the ambiguous regime the feature is for: the two RMS values within 2x of each other
        assert n_close >= 5, n_close


def test_order_follows_solver_errors_not_rms():
    """solvePnPGeneric orders the two solutions by the IPPE solver's own errors (normalised coordinates, float), not by the
    reported RMS: check both rules on many cases and require the solver-error rule to hold every time."""
    n_rms_disagree = 0
    for seed in range(5):
        for c, L in io.synthetic_cases(100 + seed, K_SYN, D_REF, kind="far"):
            ref = io.pose_hypotheses(c, K_SYN, D_REF, L)
            e0, e1 = ref["solver_err"]
            assert e0 <= e1 or abs(e0 - e1) <= 1e-6 * e1
            n_rms_disagree += int(ref["rms"][0] > ref["rms"][1])
    # informative: how often the RMS rule would have given the other order (non-zero with distortion)
    print("RMS order differs from solvePnPGeneric's order in %d cases" % n_rms_disagree)


def test_length_overrides():
    cases = io.synthetic_cases(7, K_SYN, D_REF, kind="mixed", n=24)
    lens = [0.05, 0.2, 0.3333, 0.0871]  # per-id overrides, narrowed to float like getSingleMarkerObjectPoints
    cases = [(c, lens[i % 4]) for i, (c, _) in enumerate(cases)]
    _check(cases, K_SYN, D_REF)


@pytest.mark.parametrize("D", [D_REF, D_ZERO], ids=["D_ref", "D_zero"])
def test_iterative_in_second_basin(D):
    c, L, ref = io.iterative_in_second_basin(K_SYN, D)
    got = hs_hypotheses(c[None], K_SYN, D, [L])[0]
    assert ref["iterative_match"] == 1
    swapped = io.assert_matches(got, ref)
    assert got["iterative_match"] == (0 if swapped else 1)
    assert np.abs(got["iterative_rvec"] - ref["iterative_rvec"]).max() < 1e-6  # the ITERATIVE pose it is compared with


def test_degenerate_quad_has_no_solution():
    K = K_SYN
    quads = [np.full((4, 2), 300.0, np.float32),  # all four corners on one pixel
             np.array([[300, 200], [310, 200], [320, 200], [330, 200]], np.float32)]  # on one line (no distortion)
    got = hs_hypotheses(np.array(quads), K, D_ZERO, [0.14, 0.14])
    for q, g in zip(quads, got):
        assert io.pose_hypotheses(q, K, D_ZERO, 0.14)["n"] == 0
        assert g["n"] == 0 and g["iterative_match"] == -1
        for k in ("rvec", "tvec", "rms"):
            assert np.all(np.isfinite(g[k])) and not np.any(g[k]), (k, g[k])


def test_undistort_matches_cv2():
    """The normalisation step of ippe.cuh (the one of pnp.cuh) against cv2.undistortPoints with its default criteria."""
    rng = np.random.default_rng(5)
    pts = rng.uniform([0, 0], [640, 480], (200, 2)).astype(np.float32)
    ref = cv2.undistortPoints(pts.reshape(-1, 1, 2), K_SYN, D_REF).reshape(-1, 2).astype(np.float64)
    x0 = (pts[:, 0].astype(np.float64) - K_SYN[0, 2]) / K_SYN[0, 0]
    y0 = (pts[:, 1].astype(np.float64) - K_SYN[1, 2]) / K_SYN[1, 1]
    k1, k2, p1, p2, k3 = D_REF
    x, y = x0.copy(), y0.copy()
    for _ in range(5):
        r2 = x * x + y * y
        icd = 1.0 / (1 + ((k3 * r2 + k2) * r2 + k1) * r2)
        dx = 2 * p1 * x * y + p2 * (r2 + 2 * x * x)
        dy = p1 * (r2 + 2 * y * y) + 2 * p2 * x * y
        x, y = (x0 - dx) * icd, (y0 - dy) * icd
    ours = np.stack([x, y], 1).astype(np.float32).astype(np.float64)
    assert np.abs(ours - ref).max() <= 1.2e-7 * np.abs(ref).max()  # float32 outputs: at most one ulp apart
