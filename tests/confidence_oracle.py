"""Detection with confidence: frames, cv2's detectMarkersWithConfidence with the reference parameters, and the host chain
(tests/hostsim/confidence_hostsim.cpp).  Used by tests/test_hostsim_confidence.py (CPU) and tests/test_gpu_confidence.py."""
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

METHODS = {"none": A.CORNER_REFINE_NONE, "subpix": A.CORNER_REFINE_SUBPIX, "contour": A.CORNER_REFINE_CONTOUR}


def cv2_params(method="subpix", border_bits=1, ppc=8, margin=0.13, ecr=0.6, aruco3=None):
    """The reference parameters with the ones confidence depends on replaced; aruco3 = (min_side, ratio) turns useAruco3Detection on."""
    p = ao.reference_detector_params(cornerRefinementMethod=METHODS[method], markerBorderBits=int(border_bits), perspectiveRemovePixelPerCell=int(ppc),
                                     perspectiveRemoveIgnoredMarginPerCell=float(margin), errorCorrectionRate=float(ecr))
    if aruco3 is not None:
        p.useAruco3Detection = True
        p.minSideLengthCanonicalImg = int(aruco3[0])
        p.minMarkerLengthRatioOriginalImg = float(aruco3[1])
    return p


def fid_params_for(dict_id, method="subpix", border_bits=1, ppc=8, margin=0.13, ecr=0.6):
    """The library's fid_params for the same settings."""
    from fiducials_b200 import _lib

    p = _lib.fid_params()
    _lib.load().fid_default_params(C.byref(p))
    p.dictionary = int(dict_id)
    p.cornerRefinementMethod = METHODS[method]
    p.markerBorderBits = int(border_bits)
    p.perspectiveRemovePixelPerCell = int(ppc)
    p.perspectiveRemoveIgnoredMarginPerCell = float(margin)
    p.errorCorrectionRate = float(ecr)
    return p


def cv2_detect(img, dict_id, **kw):
    """detectMarkersWithConfidence: ids [n] int32, corners [n, 4, 2] float32, confidence [n] float32, in cv2's order."""
    det = A.ArucoDetector(A.getPredefinedDictionary(dict_id), cv2_params(**kw))
    corners, ids, conf, _ = det.detectMarkersWithConfidence(img)
    if ids is None or len(ids) == 0:
        return np.zeros(0, np.int32), np.zeros((0, 4, 2), np.float32), np.zeros(0, np.float32)
    return ids.reshape(-1).astype(np.int32), np.array(corners, np.float32).reshape(-1, 4, 2), np.asarray(conf, np.float32).reshape(-1)


def _load():
    """g++ build of the harness into a temporary directory (the tree may be read-only), once per session."""
    global _harness
    if _harness is None:
        tmp = tempfile.mkdtemp(prefix="fid_conf_hostsim_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "libfid_conf_hostsim.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, os.path.join(_HERE, "hostsim", "confidence_hostsim.cpp")])
        _harness = C.CDLL(so)
        _harness.hs_detect_conf.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        _harness.hs_identify_conf.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    return _harness


def _prm(dict_id, method="subpix", border_bits=1, ppc=8, margin=0.13, ecr=0.6, border_rate=0.04):
    return np.array([dict_id, METHODS[method], border_bits, ppc, margin, ecr, border_rate], np.float64)


def host_detect(img, dict_id, **kw):
    """The host chain: ids [n], corners [n, 4, 2], confidence [n]."""
    g = np.ascontiguousarray(ao.gray(img), np.uint8)
    planes = np.ascontiguousarray(ao.threshold_planes(g), np.uint8)
    H, W = g.shape
    cap = 1024
    ids = np.zeros(cap, np.int32)
    corners = np.zeros((cap, 8), np.float32)
    conf = np.zeros(cap, np.float32)
    prm = _prm(dict_id, **kw)
    n = _load().hs_detect_conf(g.ctypes.data, planes.ctypes.data, W, H, prm.ctypes.data, ids.ctypes.data, corners.ctypes.data, conf.ctypes.data, cap)
    assert n >= 0, n
    return ids[:n].copy(), corners[:n].reshape(n, 4, 2).copy(), conf[:n].copy()


def host_identify(img, quad, dict_id, **kw):
    """(id, rotation, confidence) of one quad [4, 2] (clockwise, as the candidate stage gives it)."""
    g = np.ascontiguousarray(ao.gray(img), np.uint8)
    H, W = g.shape
    q = np.ascontiguousarray(quad, np.float32).reshape(8)
    out = np.zeros(2, np.int32)
    conf = np.zeros(1, np.float32)
    prm = _prm(dict_id, **kw)
    assert _load().hs_identify_conf(g.ctypes.data, W, H, q.ctypes.data, prm.ctypes.data, out.ctypes.data, conf.ctypes.data) == 0
    return int(out[0]), int(out[1]), float(conf[0])


# ------------------------------------------------------------------------------------------------------------------------------
# frames


def marker_frame(dict_id=A.DICT_6X6_250, marker_id=7, px=20, border_bits=1, pad=100):
    """One marker of px pixels per cell on a white frame: (gray [H, W], x0, y0, cells)."""
    d = A.getPredefinedDictionary(dict_id)
    cells = d.markerSize + 2 * border_bits
    m = A.generateImageMarker(d, int(marker_id), cells * px, borderBits=int(border_bits))
    g = np.full((cells * px + 2 * pad, cells * px + 2 * pad), 255, np.uint8)
    g[pad:pad + cells * px, pad:pad + cells * px] = m
    return g, pad, pad, cells


def paint(g, x0, y0, px, cx, cy, w=None, h=None, dx=0, dy=0):
    """Invert a w x h pixel block (default the whole cell) at offset (dx, dy) inside cell (cx, cy)."""
    w = px if w is None else w
    h = px if h is None else h
    y, x = y0 + cy * px + dy, x0 + cx * px + dx
    g[y:y + h, x:x + w] = 255 - g[y:y + h, x:x + w]
    return g


def fixed_cases():
    """(name, gray, dict_id, params, cv2 4.13's confidence with cv2's default DetectorParameters otherwise) -- DESIGN.md finding 17.
    The default perspectiveRemovePixelPerCell of cv2 is 4 (the reference runs 8)."""
    D6, D7 = A.DICT_6X6_250, A.DICT_7X7_50
    out = []
    g, x0, y0, _ = marker_frame()
    out.append(("clean", g, D6, dict(ppc=4), 1.0))
    g, x0, y0, _ = marker_frame()
    out.append(("quarter_cell", paint(g, x0, y0, 20, 3, 2, 10, 10), D6, dict(ppc=4), 0.99609375))
    g, x0, y0, _ = marker_frame()
    out.append(("one_cell", paint(g, x0, y0, 20, 3, 2), D6, dict(ppc=4), 0.984375))
    for r in range(4):
        g, x0, y0, _ = marker_frame()
        paint(g, x0, y0, 20, 3, 2)
        paint(g, x0, y0, 20, 5, 4)
        out.append(("two_cells_rot%d" % r, np.ascontiguousarray(np.rot90(g, r)), D6, dict(ppc=4), 0.96875))
    g, x0, y0, _ = marker_frame()
    out.append(("white_in_border", paint(g, x0, y0, 20, 3, 0, 10, 10, 5, 5), D6, dict(ppc=4), 0.99609375))
    g, x0, y0, _ = marker_frame(border_bits=2)
    out.append(("white_in_border_bb2", paint(g, x0, y0, 20, 4, 0, 10, 10, 5, 5), D6, dict(ppc=4, border_bits=2), 0.9975000023841858))
    g, x0, y0, _ = marker_frame(A.DICT_7X7_50, 3)
    out.append(("7x7_one_cell", paint(g, x0, y0, 20, 3, 3), D7, dict(ppc=4), 0.9876543283462524))
    g, x0, y0, _ = marker_frame()
    out.append(("strip_ppc7", paint(g, x0, y0, 20, 3, 2, 7, 20), D6, dict(ppc=7), 0.9933035969734192))
    return out


DICTS = [A.DICT_4X4_50, A.DICT_5X5_100, A.DICT_6X6_250, A.DICT_7X7_50, A.DICT_APRILTAG_36h11]
KINDS = ["clean", "blur", "noise", "bands", "occluded", "flipped"]


def render(seed, dict_id, border_bits=1, kind="clean", W=640, H=480, n_markers=6):
    """A gray frame [H, W] with n_markers markers of dict_id (random id, size, quarter turn, mild perspective) in a grid of cells,
    then by kind: blurred, noisy, under gray bands of another brightness, partly covered by a gray blob, or with inner cells
    inverted so that they decode only through error correction (some beyond it)."""
    rng = np.random.default_rng(seed)
    d = A.getPredefinedDictionary(dict_id)
    cells = d.markerSize + 2 * border_bits
    n_ids = min(d.bytesList.shape[0], 250)
    g = np.full((H, W), int(rng.integers(170, 240)), np.uint8)
    cols = int(np.ceil(np.sqrt(n_markers * W / H)))
    rows = int(np.ceil(n_markers / cols))
    cw, ch = W // cols, H // rows
    for cell in rng.permutation(rows * cols)[:n_markers]:
        r, c = divmod(int(cell), cols)
        px = int(rng.integers(max(3, 40 // cells), max(4, int(0.8 * min(cw, ch)) // cells) + 1))
        side = cells * px
        m = A.generateImageMarker(d, int(rng.integers(n_ids)), side, borderBits=int(border_bits))
        if kind == "flipped":  # whole inner cells inverted
            for _ in range(int(rng.integers(1, 4))):
                cx, cy = (int(v) for v in rng.integers(border_bits, cells - border_bits, 2))
                m[cy * px:(cy + 1) * px, cx * px:(cx + 1) * px] = 255 - m[cy * px:(cy + 1) * px, cx * px:(cx + 1) * px]
        m = np.ascontiguousarray(np.rot90(m, int(rng.integers(4))))
        pad = max(4, side // 5)
        ts = side + 2 * pad
        if ts > min(cw, ch):
            continue
        tile = np.full((ts, ts), 255, np.uint8)
        tile[pad:pad + side, pad:pad + side] = m
        src = np.float32([[0, 0], [ts, 0], [ts, ts], [0, ts]])
        dst = src + np.float32(rng.uniform(0, 0.12 * ts, (4, 2))) * np.float32([[1, 1], [-1, 1], [-1, -1], [1, -1]])
        tile = cv2.warpPerspective(tile, cv2.getPerspectiveTransform(src, dst), (ts, ts), flags=cv2.INTER_LINEAR, borderValue=255)
        y0 = r * ch + int(rng.integers(0, ch - ts + 1))
        x0 = c * cw + int(rng.integers(0, cw - ts + 1))
        g[y0:y0 + ts, x0:x0 + ts] = np.minimum(g[y0:y0 + ts, x0:x0 + ts], tile)
        if kind == "occluded":  # a gray blob over part of the marker
            oy, ox = (int(v) for v in rng.integers(pad, pad + side - px, 2))
            rad = int(rng.integers(px // 2 + 1, 2 * px + 2))
            cv2.circle(g, (x0 + ox, y0 + oy), rad, int(rng.integers(60, 200)), -1)
    if kind == "bands":  # brightness bands across the frame
        for _ in range(3):
            y = int(rng.integers(0, H - 20))
            h = int(rng.integers(10, 60))
            g[y:y + h] = np.clip(g[y:y + h].astype(np.int32) + int(rng.integers(-60, 40)), 0, 255).astype(np.uint8)
    if kind == "blur":
        g = cv2.GaussianBlur(g, (0, 0), float(rng.uniform(0.8, 2.0)))
    noise = 8.0 if kind == "noise" else 2.0
    g = np.clip(g + rng.normal(0, noise, g.shape), 0, 255).astype(np.uint8)
    return g


def sweep_cases(n=180):
    """(name, gray, dict_id, params) of the seeded sweep: every dictionary, markerBorderBits 1 and 2, perspectiveRemovePixelPerCell
    4 / 7 / 8 with the default and a larger margin, the three refinement methods and every kind of frame."""
    ppcs = [(4, 0.13), (7, 0.13), (8, 0.13), (4, 0.3), (7, 0.25), (8, 0.3)]
    methods = ["none", "subpix", "contour"]
    for i in range(n):
        dict_id = DICTS[i % len(DICTS)]
        bb = 1 + (i // len(DICTS)) % 2
        ppc, margin = ppcs[(i // 3) % len(ppcs)]
        method = methods[i % 3]
        kind = KINDS[(i // 2) % len(KINDS)]
        if (A.getPredefinedDictionary(dict_id).markerSize + 2 * bb) * ppc > 72:  # the library's largest canonical image (FID_MAX_WARP_SIDE)
            ppc = 4
        kw = dict(method=method, border_bits=bb, ppc=ppc, margin=margin)
        yield "%d/d%d/bb%d/ppc%d/m%g/%s/%s" % (i, dict_id, bb, ppc, margin, method, kind), render(9000 + i, dict_id, bb, kind), dict_id, kw
