"""Detection with detectInvertedMarker (DESIGN.md finding 18): frames, cv2 4.13's detectMarkers / detectMarkersWithConfidence with the
reference parameters and the flag, and the host chain (tests/hostsim/inverted_hostsim.cpp).  Used by tests/test_hostsim_inverted.py
(CPU) and tests/test_gpu_inverted.py."""
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


def cv2_params(inverted=True, method="subpix", border_bits=1, ppc=8, margin=0.13, ecr=0.6, aruco3=None):
    """The reference parameters with detectInvertedMarker and the ones the sweep varies; aruco3 = (min_side, ratio) turns
    useAruco3Detection on."""
    p = ao.reference_detector_params(cornerRefinementMethod=METHODS[method], markerBorderBits=int(border_bits), perspectiveRemovePixelPerCell=int(ppc),
                                     perspectiveRemoveIgnoredMarginPerCell=float(margin), errorCorrectionRate=float(ecr))
    p.detectInvertedMarker = bool(inverted)
    if aruco3 is not None:
        p.useAruco3Detection = True
        p.minSideLengthCanonicalImg = int(aruco3[0])
        p.minMarkerLengthRatioOriginalImg = float(aruco3[1])
    return p


def fid_params_for(dict_id, method="subpix", border_bits=1, ppc=8, margin=0.13, ecr=0.6):
    """The library's fid_params for the same settings (the flag itself is fid_set_detect_inverted_marker)."""
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


def _out(corners, ids, conf=None):
    if ids is None or len(ids) == 0:
        e = (np.zeros(0, np.int32), np.zeros((0, 4, 2), np.float32))
        return e + ((np.zeros(0, np.float32),) if conf is not None else ())
    r = (ids.reshape(-1).astype(np.int32), np.array(corners, np.float32).reshape(-1, 4, 2))
    return r + ((np.asarray(conf, np.float32).reshape(-1),) if conf is not None else ())


def cv2_detect(img, dict_id, inverted=True, **kw):
    """detectMarkers: ids [n] int32, corners [n, 4, 2] float32 in cv2's order, and the number of rejected candidates."""
    det = A.ArucoDetector(A.getPredefinedDictionary(dict_id), cv2_params(inverted, **kw))
    corners, ids, rej = det.detectMarkers(img)
    return _out(corners, ids) + (len(rej),)


def cv2_detect_conf(img, dict_id, inverted=True, **kw):
    """detectMarkersWithConfidence: ids, corners, confidence [n] float32."""
    det = A.ArucoDetector(A.getPredefinedDictionary(dict_id), cv2_params(inverted, **kw))
    corners, ids, conf, _ = det.detectMarkersWithConfidence(img)
    return _out(corners, ids, conf)


def _load():
    """g++ build of the harness into a temporary directory (the tree may be read-only), once per session."""
    global _harness
    if _harness is None:
        tmp = tempfile.mkdtemp(prefix="fid_inv_hostsim_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "libfid_inv_hostsim.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, os.path.join(_HERE, "hostsim", "inverted_hostsim.cpp")])
        _harness = C.CDLL(so)
        _harness.hs_detect_inv.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        _harness.hs_identify_inv.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    return _harness


def _prm(dict_id, method="subpix", border_bits=1, ppc=8, margin=0.13, ecr=0.6, border_rate=0.04):
    return np.array([dict_id, METHODS[method], border_bits, ppc, margin, ecr, border_rate], np.float64)


def host_detect(img, dict_id, inverted=True, **kw):
    """The host chain: ids [n], corners [n, 4, 2], confidence [n], polarity [n] (1 = white marker)."""
    g = np.ascontiguousarray(ao.gray(img), np.uint8)
    planes = np.ascontiguousarray(ao.threshold_planes(g), np.uint8)
    H, W = g.shape
    cap = 1024
    ids = np.zeros(cap, np.int32)
    corners = np.zeros((cap, 8), np.float32)
    conf = np.zeros(cap, np.float32)
    pol = np.zeros(cap, np.int32)
    prm = _prm(dict_id, **kw)
    n = _load().hs_detect_inv(g.ctypes.data, planes.ctypes.data, W, H, prm.ctypes.data, int(bool(inverted)), ids.ctypes.data, corners.ctypes.data, conf.ctypes.data,
                              pol.ctypes.data, cap)
    assert n >= 0, n
    return ids[:n].copy(), corners[:n].reshape(n, 4, 2).copy(), conf[:n].copy(), pol[:n].copy()


def host_identify(img, quad, dict_id, inverted=True, **kw):
    """(id, rotation, polarity, confidence) of one quad [4, 2] (clockwise, as the candidate stage gives it)."""
    g = np.ascontiguousarray(ao.gray(img), np.uint8)
    H, W = g.shape
    q = np.ascontiguousarray(quad, np.float32).reshape(8)
    out = np.zeros(3, np.int32)
    conf = np.zeros(1, np.float32)
    prm = _prm(dict_id, **kw)
    assert _load().hs_identify_inv(g.ctypes.data, W, H, q.ctypes.data, prm.ctypes.data, int(bool(inverted)), out.ctypes.data, conf.ctypes.data) == 0
    return int(out[0]), int(out[1]), int(out[2]), float(conf[0])


# ------------------------------------------------------------------------------------------------------------------------------
# frames

DICTS = [A.DICT_4X4_50, A.DICT_5X5_1000, A.DICT_6X6_250, A.DICT_7X7_50, A.DICT_APRILTAG_36h11, A.DICT_ARUCO_ORIGINAL]
KINDS = ["clean", "blur", "noise", "oblique", "nested"]
POLARITIES = ["normal", "inverted", "mixed"]
SIZES = [(640, 480), (1280, 720), (1920, 1080)]


def lone_marker(px=15, dict_id=A.DICT_6X6_250, marker_id=7, pad=50, white=False):
    """One marker of px pixels per cell at (pad, pad) on a frame of 2 pad + side; white: the whole frame inverted."""
    d = A.getPredefinedDictionary(dict_id)
    side = (d.markerSize + 2) * px
    g = np.full((side + 2 * pad, side + 2 * pad), 255, np.uint8)
    g[pad:pad + side, pad:pad + side] = A.generateImageMarker(d, int(marker_id), side)
    return 255 - g if white else g


def render(seed, dict_id, border_bits=1, kind="clean", polarity="normal", W=640, H=480, n_markers=6):
    """A gray frame [H, W] with n_markers markers of dict_id (random id, size, quarter turn, mild perspective, each on a light quiet
    zone) in a grid of cells.  polarity: "inverted" inverts the whole frame, "mixed" the tile of every other marker (a white marker
    on a dark plate).  kind: blurred, noisy, strongly oblique, or "nested" (the first marker's quiet zone holds a smaller marker of
    the other polarity inside the first's tile, as a marker printed on a plate that carries another)."""
    rng = np.random.default_rng(seed)
    d = A.getPredefinedDictionary(dict_id)
    cells = d.markerSize + 2 * border_bits
    n_ids = min(d.bytesList.shape[0], 250)
    g = np.full((H, W), int(rng.integers(150, 240)), np.uint8)
    cols = int(np.ceil(np.sqrt(n_markers * W / H)))
    rows = int(np.ceil(n_markers / cols))
    cw, ch = W // cols, H // rows
    persp = 0.3 if kind == "oblique" else 0.12
    for k, cell in enumerate(rng.permutation(rows * cols)[:n_markers]):
        r, c = divmod(int(cell), cols)
        px = int(rng.integers(max(3, 40 // cells), max(4, int(0.7 * min(cw, ch)) // cells) + 1))
        side = cells * px
        m = A.generateImageMarker(d, int(rng.integers(n_ids)), side, borderBits=int(border_bits))
        m = np.ascontiguousarray(np.rot90(m, int(rng.integers(4))))
        pad = max(4, side // 5)
        ts = side + 2 * pad
        if ts > min(cw, ch):
            continue
        tile = np.full((ts, ts), 255, np.uint8)
        tile[pad:pad + side, pad:pad + side] = m
        if kind == "nested" and k == 0 and px >= 6:  # a small marker of the other polarity in the quiet zone's corner
            sp = max(2, pad // (cells + 2))
            ss = cells * sp
            if ss + 2 <= pad:
                sm = 255 - A.generateImageMarker(d, int(rng.integers(n_ids)), ss, borderBits=int(border_bits))
                tile[1:1 + ss, 1:1 + ss] = sm
        if polarity == "mixed" and k % 2 == 1:
            tile = 255 - tile
        src = np.float32([[0, 0], [ts, 0], [ts, ts], [0, ts]])
        dst = src + np.float32(rng.uniform(0, persp * ts, (4, 2))) * np.float32([[1, 1], [-1, 1], [-1, -1], [1, -1]])
        M = cv2.getPerspectiveTransform(src, dst)
        tile = cv2.warpPerspective(tile, M, (ts, ts), flags=cv2.INTER_LINEAR, borderValue=0)
        mask = cv2.warpPerspective(np.full((ts, ts), 255, np.uint8), M, (ts, ts), flags=cv2.INTER_NEAREST, borderValue=0)
        y0 = r * ch + int(rng.integers(0, ch - ts + 1))
        x0 = c * cw + int(rng.integers(0, cw - ts + 1))
        reg = g[y0:y0 + ts, x0:x0 + ts]
        reg[mask > 0] = tile[mask > 0]
    if kind == "blur":
        g = cv2.GaussianBlur(g, (0, 0), float(rng.uniform(0.8, 2.0)))
    noise = 8.0 if kind == "noise" else 2.0
    g = np.clip(g + rng.normal(0, noise, g.shape), 0, 255).astype(np.uint8)
    if polarity == "inverted":
        g = 255 - g
    return g


def sweep_cases(n=120):
    """(name, gray, dict_id, params) of the seeded sweep: every dictionary, markerBorderBits 1 and 2, the three refinement methods,
    the three polarities, every kind of frame and three frame sizes; ppc 4 where the canonical image would exceed the library's
    largest (FID_MAX_WARP_SIDE)."""
    methods = ["none", "subpix", "contour"]
    for i in range(n):
        dict_id = DICTS[i % len(DICTS)]
        bb = 1 + (i // len(DICTS)) % 2
        method = methods[i % 3]
        pol = POLARITIES[(i // 2) % 3]
        kind = KINDS[(i // 3) % len(KINDS)]
        W, H = SIZES[(i // 5) % len(SIZES)] if i % 4 == 0 else SIZES[0]
        ppc = 8 if (A.getPredefinedDictionary(dict_id).markerSize + 2 * bb) * 8 <= 72 else 4
        kw = dict(method=method, border_bits=bb, ppc=ppc)
        yield "%d/d%d/bb%d/%s/%s/%s/%dx%d" % (i, dict_id, bb, method, pol, kind, W, H), render(7000 + i, dict_id, bb, kind, pol, W, H), dict_id, kw


def blank_frames():
    """Frames without markers: flat, noise, and a dark and a light square (no code)."""
    rng = np.random.default_rng(5)
    out = [("flat", np.full((480, 640), 200, np.uint8)), ("noise", rng.integers(0, 256, (480, 640)).astype(np.uint8))]
    g = np.full((480, 640), 220, np.uint8)
    g[100:220, 100:220] = 20
    out.append(("dark_square", g))
    out.append(("light_square", 255 - g))
    return out
