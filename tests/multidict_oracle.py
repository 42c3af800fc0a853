"""Detection with several dictionaries: frames with markers of several families, cv2's detectMarkersMultiDict with the reference
parameters, and the host chain (tests/hostsim/multidict_hostsim.cpp).  Used by tests/test_hostsim_multidict.py (CPU) and
tests/test_gpu_multidict.py."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import cv2
import numpy as np

from oracle import aruco_oracle as ao

A = cv2.aruco
_HERE = os.path.dirname(os.path.abspath(__file__))
_harness = None

# the dictionary lists of the sweep: different marker sizes, one size from two families, overlapping dictionaries, a repeated entry
DICT_LISTS = {
    "sizes_4_6_5": [A.DICT_4X4_50, A.DICT_6X6_250, A.DICT_5X5_1000],
    "6x6_36h11": [A.DICT_6X6_250, A.DICT_APRILTAG_36h11],
    "5x5_25h9": [A.DICT_5X5_100, A.DICT_APRILTAG_25h9],
    "overlap_6x6": [A.DICT_6X6_250, A.DICT_6X6_1000],
    "repeated": [A.DICT_4X4_50, A.DICT_4X4_50],
    "original_mip": [A.DICT_ARUCO_ORIGINAL, A.DICT_ARUCO_MIP_36h12, A.DICT_4X4_100],
    "four": [A.DICT_6X6_250, A.DICT_APRILTAG_36h11, A.DICT_4X4_50, A.DICT_5X5_1000],
}


def _marker(dict_id, marker_id, side):
    return A.generateImageMarker(A.getPredefinedDictionary(dict_id), int(marker_id), int(side), borderBits=1)


def render_mixed(W, H, dict_ids, seed, n_markers=8, nested=False, noise=3.0):
    """A gray-on-BGR frame [H, W, 3] with n_markers markers drawn from the families in dict_ids (random family, id, size, quarter
    turn), the whole frame under a mild random perspective warp, blurred and with noise.  nested: one marker of the second family
    drawn inside a white cell of a big marker of the first."""
    rng = np.random.default_rng(seed)
    g = np.full((H, W), 200, np.uint8)
    cols = max(1, int(np.ceil(np.sqrt(n_markers * W / H))))
    rows = max(1, int(np.ceil(n_markers / cols)))
    cw, ch = W // cols, H // rows
    cells = rng.permutation(rows * cols)[:n_markers]
    for k, cell in enumerate(cells):
        r, c = divmod(int(cell), cols)
        d = dict_ids[int(rng.integers(len(dict_ids)))] if not (nested and k == 0) else dict_ids[0]
        n_ids = A.getPredefinedDictionary(d).bytesList.shape[0]
        side = int(rng.uniform(0.45, 0.85) * min(cw, ch))
        if nested and k == 0:  # big enough that a cell holds a detectable marker
            side = int(0.95 * min(cw, ch))
        m = np.rot90(_marker(d, rng.integers(min(n_ids, 250)), side), int(rng.integers(4)))
        if nested and k == 0:  # a second-family marker inside the first white cell of this marker
            ms = A.getPredefinedDictionary(d).markerSize + 2
            cs = side // ms
            m = np.ascontiguousarray(m)
            for yy in range(1, ms - 1):
                hit = [xx for xx in range(1, ms - 1) if m[yy * cs + cs // 2, xx * cs + cs // 2] > 127 and cs >= 24]
                if hit:
                    xx = hit[0]
                    inner = _marker(dict_ids[1], rng.integers(20), cs * 2 // 3)
                    o = (cs - inner.shape[0]) // 2
                    m[yy * cs + o:yy * cs + o + inner.shape[0], xx * cs + o:xx * cs + o + inner.shape[1]] = inner
                    break
        y0 = r * ch + int(rng.integers(0, ch - side + 1))
        x0 = c * cw + int(rng.integers(0, cw - side + 1))
        g[y0:y0 + side, x0:x0 + side] = m
    Hm = np.array([[1 + rng.uniform(-0.03, 0.03), rng.uniform(-0.05, 0.05), rng.uniform(-5, 5)],
                   [rng.uniform(-0.05, 0.05), 1 + rng.uniform(-0.03, 0.03), rng.uniform(-5, 5)],
                   [rng.uniform(-2e-5, 2e-5), rng.uniform(-2e-5, 2e-5), 1.0]])
    g = cv2.warpPerspective(g, Hm, (W, H), flags=cv2.INTER_LINEAR, borderValue=200)
    g = cv2.GaussianBlur(g, (3, 3), 0.7)
    g = np.clip(g + rng.normal(0, noise, g.shape), 0, 255).astype(np.uint8)
    return np.ascontiguousarray(cv2.cvtColor(g, cv2.COLOR_GRAY2BGR))


def blank_frame(W, H, seed, noise_only=False):
    rng = np.random.default_rng(seed)
    g = rng.integers(0, 256, (H, W)).astype(np.uint8) if noise_only else np.full((H, W), int(rng.integers(0, 256)), np.uint8)
    return np.ascontiguousarray(cv2.cvtColor(g, cv2.COLOR_GRAY2BGR))


def cv2_multi(bgr, dict_ids, method=1):
    """detectMarkersMultiDict with the reference parameters: ids [n], corners [n, 4, 2] float32, dict indices [n], rejected [m, 4, 2]."""
    p = ao.reference_detector_params(cornerRefinementMethod=method)
    det = A.ArucoDetector(A.getPredefinedDictionary(dict_ids[0]), p)
    det.setDictionaries([A.getPredefinedDictionary(d) for d in dict_ids])
    corners, ids, rej, di = det.detectMarkersMultiDict(bgr)
    n = 0 if ids is None else len(ids)
    ids = np.zeros(0, np.int32) if ids is None else ids.reshape(-1).astype(np.int32)
    di = np.zeros(0, np.int32) if di is None or n == 0 else np.asarray(di).reshape(-1).astype(np.int32)
    return ids, np.array(corners, np.float32).reshape(-1, 4, 2), di, np.array(rej, np.float32).reshape(-1, 4, 2)


def cv2_single(bgr, dict_id, method=1):
    det = A.ArucoDetector(A.getPredefinedDictionary(dict_id), ao.reference_detector_params(cornerRefinementMethod=method))
    corners, ids, rej = det.detectMarkers(bgr)
    ids = np.zeros(0, np.int32) if ids is None else ids.reshape(-1).astype(np.int32)
    return ids, np.array(corners, np.float32).reshape(-1, 4, 2), np.array(rej, np.float32).reshape(-1, 4, 2)


def _load():
    """g++ build of the harness into a temporary directory (the tree may be read-only), once per session."""
    global _harness
    if _harness is None:
        tmp = tempfile.mkdtemp(prefix="fid_multidict_hostsim_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "libfid_multidict_hostsim.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, os.path.join(_HERE, "hostsim", "multidict_hostsim.cpp")])
        _harness = C.CDLL(so)
    return _harness


def host_multi(bgr, dict_ids, method=1):
    """The host chain: ids [n], corners [n, 4, 2], dict indices [n]."""
    g = np.ascontiguousarray(ao.gray(bgr))
    planes = np.ascontiguousarray(ao.threshold_planes(g), np.uint8)
    H, W = g.shape
    cap = 1024
    ids = np.zeros(cap, np.int32)
    corners = np.zeros((cap, 8), np.float32)
    di = np.zeros(cap, np.int32)
    dl = np.ascontiguousarray(dict_ids, np.int32)
    vp = C.c_void_p
    n = _load().hs_detect_multi(g.ctypes.data_as(vp), planes.ctypes.data_as(vp), W, H, len(dl), dl.ctypes.data_as(vp), int(method), ids.ctypes.data_as(vp),
                                corners.ctypes.data_as(vp), di.ctypes.data_as(vp), cap)
    assert n >= 0, n
    return ids[:n].copy(), corners[:n].reshape(n, 4, 2).copy(), di[:n].copy()


def sweep_cases(n_frames=160):
    """(name, bgr, dict_ids, method) of the seeded sweep: every dictionary list, NONE / SUBPIX / CONTOUR, 640x480 and 1280x720, nested
    markers, blank and noise frames."""
    names = list(DICT_LISTS)
    for i in range(n_frames):
        key = names[i % len(names)]
        dl = DICT_LISTS[key]
        method = (i // len(names)) % 3
        if i % 23 == 22:
            yield "blank/%d" % i, blank_frame(640, 480, i), dl, method
            continue
        if i % 29 == 28:
            yield "noise/%d" % i, blank_frame(320, 240, i, noise_only=True), dl, method
            continue
        W, H = (1280, 720) if i % 5 == 0 else (640, 480)
        nested = i % 7 == 3
        yield "%s/%d/m%d%s" % (key, i, method, "/nested" if nested else ""), render_mixed(W, H, dl, 1000 + i, n_markers=8 if W == 640 else 14, nested=nested), dl, method
