"""Detection with useAruco3Detection: frames, cv2's ArucoDetector with the reference parameters plus the mode, the planes cv2 builds
(cv2.resize, repeated cv2.pyrDown) and the host chain (tests/hostsim/aruco3_hostsim.cpp).  Used by tests/test_hostsim_aruco3.py (CPU)
and tests/test_gpu_aruco3.py."""
import atexit
import ctypes as C
import math
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


def params(min_side=32, ratio=0.02, **overrides):
    p = ao.reference_detector_params(**overrides)
    p.useAruco3Detection = True
    p.minSideLengthCanonicalImg = int(min_side)
    p.minMarkerLengthRatioOriginalImg = float(ratio)
    return p


def cv2_detect(bgr, dict_id, min_side=32, ratio=0.02, **overrides):
    """detectMarkers with the mode on: ids [n] int32, corners [n, 4, 2] float32, in cv2's order."""
    det = A.ArucoDetector(A.getPredefinedDictionary(dict_id), params(min_side, ratio, **overrides))
    corners, ids, _ = det.detectMarkers(bgr)
    ids = np.zeros(0, np.int32) if ids is None else ids.reshape(-1).astype(np.int32)
    return ids, np.array(corners, np.float32).reshape(-1, 4, 2)


def geometry(W, H, min_side, ratio):
    """cv2's step 0 / 1.1 in float32: (seg_w, seg_h, n_levels including level 0, closest)."""
    f32 = np.float32
    fxfy = f32(min_side) / (f32(min_side) + f32(max(W, H)) * f32(ratio))
    area = f32(W * H)
    num_levels = int(math.log2(float(area / f32(min_side * min_side))) / 2.0)
    closest = int(np.rint(math.log2(float(area / (area * fxfy * fxfy))) / 2.0))
    if fxfy == f32(1):
        return W, H, num_levels + 1, closest
    return int(np.rint(fxfy * f32(W))), int(np.rint(fxfy * f32(H))), num_levels + 1, closest


def cv2_planes(gray, min_side, ratio):
    """(segmentation plane, [pyramid levels 0..]) as cv2.resize and repeated cv2.pyrDown make them."""
    H, W = gray.shape
    sw, sh, n_levels, _ = geometry(W, H, min_side, ratio)
    seg = gray if (sw, sh) == (W, H) else cv2.resize(gray, (sw, sh), interpolation=cv2.INTER_LINEAR)
    pyr = [gray]
    for _ in range(n_levels - 1):
        pyr.append(cv2.pyrDown(pyr[-1]))
    return seg, pyr


def _load():
    """g++ build of the harness into a temporary directory (the tree may be read-only), once per session."""
    global _harness
    if _harness is None:
        tmp = tempfile.mkdtemp(prefix="fid_aruco3_hostsim_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "libfid_aruco3_hostsim.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, os.path.join(_HERE, "hostsim", "aruco3_hostsim.cpp")])
        _harness = C.CDLL(so)
        _harness.hs_a3_planes.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]
        _harness.hs_a3_level_for.argtypes = [C.c_int, C.c_int, C.c_int, C.c_double, C.c_int]
        _harness.hs_detect_aruco3.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_void_p, C.c_void_p, C.c_int]
    return _harness


def host_planes(gray, min_side, ratio):
    """The host build's (segmentation plane, [pyramid levels 0..], closest)."""
    g = np.ascontiguousarray(gray, np.uint8)
    H, W = g.shape
    info = np.zeros(4, np.int32)
    assert _load().hs_a3_planes(g.ctypes.data, W, H, int(min_side), float(ratio), info.ctypes.data, None, None) == 0
    sw, sh, n_levels, closest = (int(v) for v in info)
    seg = np.zeros((sh, sw), np.uint8)
    sizes, w, h = [], W, H
    for _ in range(n_levels):
        sizes.append((h, w))
        w, h = (w + 1) // 2, (h + 1) // 2
    pyr = np.zeros(sum(a * b for a, b in sizes[1:]) + 1, np.uint8)
    _load().hs_a3_planes(g.ctypes.data, W, H, int(min_side), float(ratio), info.ctypes.data, seg.ctypes.data, pyr.ctypes.data)
    levels, off = [g], 0
    for h, w in sizes[1:]:
        levels.append(pyr[off:off + h * w].reshape(h, w))
        off += h * w
    return seg, levels, closest


def host_level_for(W, H, min_side, ratio, contour_len):
    return _load().hs_a3_level_for(W, H, int(min_side), float(ratio), int(contour_len))


def host_detect(bgr, dict_id, min_side=32, ratio=0.02):
    """The host chain: ids [n], corners [n, 4, 2] at full resolution."""
    g = np.ascontiguousarray(ao.gray(bgr) if bgr.ndim == 3 else bgr)
    seg, _, _ = host_planes(g, min_side, ratio)
    planes = np.ascontiguousarray(ao.threshold_planes(seg), np.uint8)
    H, W = g.shape
    cap = 1024
    ids = np.zeros(cap, np.int32)
    corners = np.zeros((cap, 8), np.float32)
    n = _load().hs_detect_aruco3(g.ctypes.data, W, H, planes.ctypes.data, int(dict_id), int(min_side), float(ratio), ids.ctypes.data, corners.ctypes.data, cap)
    assert n >= 0, n
    return ids[:n].copy(), corners[:n].reshape(n, 4, 2).copy()


def _marker(dict_id, marker_id, side):
    return A.generateImageMarker(A.getPredefinedDictionary(dict_id), int(marker_id), int(side), borderBits=1)


def render(W, H, dict_id, seed, n_markers=8, side_range=(0.3, 0.85), oblique=0.0, corners_first=False, blur=0.7, noise=3.0):
    """A gray-on-BGR frame [H, W, 3]: n_markers markers of dict_id in a grid of cells (random id, size within side_range of the
    cell, quarter turn), each under its own perspective warp of strength `oblique`, optionally the first four in the frame
    corners; blurred with sigma `blur` and noise added."""
    rng = np.random.default_rng(seed)
    g = np.full((H, W), int(rng.integers(150, 230)), np.uint8)
    cols = max(1, int(np.ceil(np.sqrt(n_markers * W / H))))
    rows = max(1, int(np.ceil(n_markers / cols)))
    cw, ch = W // cols, H // rows
    cells = list(rng.permutation(rows * cols)[:n_markers])
    if corners_first and rows > 1 and cols > 1:
        corner_cells = [0, cols - 1, (rows - 1) * cols, rows * cols - 1]
        cells = corner_cells + [c for c in cells if c not in corner_cells][:max(0, n_markers - 4)]
    n_ids = A.getPredefinedDictionary(dict_id).bytesList.shape[0]
    for cell in cells:
        r, c = divmod(int(cell), cols)
        side = max(8, int(rng.uniform(*side_range) * min(cw, ch)))
        m = np.rot90(_marker(dict_id, rng.integers(min(n_ids, 250)), side), int(rng.integers(4)))
        pad = side // 6 + 2
        tile = np.full((side + 2 * pad, side + 2 * pad), 255, np.uint8)
        tile[pad:pad + side, pad:pad + side] = m
        ts = tile.shape[0]
        if oblique > 0:
            d = oblique * ts
            src = np.float32([[0, 0], [ts, 0], [ts, ts], [0, ts]])
            dst = src + np.float32(rng.uniform(0, d, (4, 2))) * np.float32([[1, 1], [-1, 1], [-1, -1], [1, -1]])
            tile = cv2.warpPerspective(tile, cv2.getPerspectiveTransform(src, dst), (ts, ts), flags=cv2.INTER_LINEAR, borderValue=255)
        if ts > min(cw, ch):
            continue
        y0 = r * ch + int(rng.integers(0, ch - ts + 1))
        x0 = c * cw + int(rng.integers(0, cw - ts + 1))
        if corners_first and cell in (0, cols - 1, (rows - 1) * cols, rows * cols - 1):  # hug the frame corner
            y0 = r * ch + (2 if r == 0 else ch - ts - 2)
            x0 = c * cw + (2 if c == 0 else cw - ts - 2)
        g[y0:y0 + ts, x0:x0 + ts] = np.minimum(g[y0:y0 + ts, x0:x0 + ts], tile)
    if blur > 0:
        g = cv2.GaussianBlur(g, (0, 0), blur)
    g = np.clip(g + rng.normal(0, noise, g.shape), 0, 255).astype(np.uint8)
    return np.ascontiguousarray(cv2.cvtColor(g, cv2.COLOR_GRAY2BGR))


def blank_frame(W, H, seed, noise_only=False):
    rng = np.random.default_rng(seed)
    g = rng.integers(0, 256, (H, W)).astype(np.uint8) if noise_only else np.full((H, W), int(rng.integers(0, 256)), np.uint8)
    return np.ascontiguousarray(cv2.cvtColor(g, cv2.COLOR_GRAY2BGR))


SIZES = [(640, 480), (1280, 720), (1920, 1080), (3840, 2160)]
RATIOS = [0.0, 0.01, 0.02, 0.05]
MIN_SIDES = [16, 32, 64]
DICTS = [A.DICT_6X6_250, A.DICT_APRILTAG_36h11, A.DICT_4X4_50]
KINDS = ["near_min", "large", "oblique", "corners", "blurred"]


def sweep_cases(n_frames=160):
    """(name, bgr, dict_id, min_side, ratio) of the seeded sweep: every size, ratio, minSide, dictionary and kind of marker, with
    blank and noise frames."""
    for i in range(n_frames):
        W, H = SIZES[i % len(SIZES)]
        ratio = RATIOS[(i // len(SIZES)) % len(RATIOS)]
        min_side = MIN_SIDES[(i // 16) % len(MIN_SIDES)]
        dict_id = DICTS[i % len(DICTS)]
        kind = KINDS[(i // 3) % len(KINDS)]
        if i % 23 == 22:
            yield "blank/%d" % i, blank_frame(W, H, i), dict_id, min_side, ratio
            continue
        if i % 29 == 28:
            yield "noise/%d" % i, blank_frame(W, H, i, noise_only=True), dict_id, min_side, ratio
            continue
        seed = 5000 + i
        n = 12 if W >= 1920 else 8
        if kind == "near_min":  # markers a little above minSide in the segmentation plane, and some below
            sw = geometry(W, H, min_side, ratio)[0]
            target = min_side * W / sw  # full-resolution side that maps to minSide
            cell = min(W / math.ceil(math.sqrt(n * W / H)), H / math.ceil(n / math.ceil(math.sqrt(n * W / H))))
            lo, hi = 0.8 * target / cell, 1.6 * target / cell
            lo, hi = min(lo, 0.8), min(max(hi, lo + 0.05), 0.85)
            bgr = render(W, H, dict_id, seed, n, side_range=(lo, hi))
        elif kind == "large":
            bgr = render(W, H, dict_id, seed, 4, side_range=(0.6, 0.8))
        elif kind == "oblique":
            bgr = render(W, H, dict_id, seed, n, side_range=(0.4, 0.8), oblique=0.22)
        elif kind == "corners":
            bgr = render(W, H, dict_id, seed, n, side_range=(0.4, 0.7), corners_first=True)
        else:
            bgr = render(W, H, dict_id, seed, n, side_range=(0.3, 0.8), blur=2.0)
        yield "%s/%d/%dx%d/r%g/s%d" % (kind, i, W, H, ratio, min_side), bgr, dict_id, min_side, ratio
