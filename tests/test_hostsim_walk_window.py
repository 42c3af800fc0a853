"""The register window the border walk's hot loops keep over the walker's halo tile (TileWin, contour_walk.cuh) and the
grouped point stores of trace_segment, on the host build of the same code: the window must show HaloView::idx9 of the
walker's pixel after every step, whatever tile edge the step crosses, and a segment must write exactly its own words."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

_HERE = os.path.dirname(os.path.abspath(__file__))
_harness = None


def _load():
    """g++ build of the harness into a temporary directory (the tree may be read-only), once per session."""
    global _harness
    if _harness is None:
        tmp = tempfile.mkdtemp(prefix="fid_walk_window_hostsim_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "libfid_walk_window_hostsim.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, os.path.join(_HERE, "hostsim", "walk_window_hostsim.cpp")])
        _harness = C.CDLL(so)
    return _harness


def _window_check(plane, max_steps=400):
    lib = _load()
    lib.hs_window_check.restype = C.c_int
    lib.hs_window_check.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
    plane = np.ascontiguousarray(plane, np.uint8)
    out = np.zeros(2, np.int64)
    bad = lib.hs_window_check(plane.ctypes.data, plane.shape[1], plane.shape[0], max_steps, out.ctypes.data)
    return bad, int(out[0]), int(out[1])


def _segment_check(plane, ck_step):
    lib = _load()
    lib.hs_trace_segment_check.restype = C.c_int
    lib.hs_trace_segment_check.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
    plane = np.ascontiguousarray(plane, np.uint8)
    out = np.zeros(6, np.int64)
    bad = lib.hs_trace_segment_check(plane.ctypes.data, plane.shape[1], plane.shape[0], ck_step, out.ctypes.data)
    return bad, out


def _edge_plane(W, H):
    """Borders that run along and across the 30-pixel tile edges and the image edge: bars whose sides lie on rows / columns
    0, 29 and 30 mod 30, a frame on the image edge, a staircase and a zigzag over the tile corners, a blob in the last tile."""
    p = np.zeros((H, W), np.uint8)
    p[0, :] = p[H - 1, :] = p[:, 0] = p[:, W - 1] = 1
    for y0 in range(29, H - 3, 30):
        p[y0:y0 + 2, 3:W - 3] = 1       # rows 29 and 30 mod 30: the bar's two sides lie in different tile rows
    for x0 in range(59, W - 3, 60):
        p[3:H - 3, x0:x0 + 2] = 1
    for k in range(min(W, H) - 8):       # diagonal staircase through the tile corners
        p[4 + k, 4 + k:6 + k] = 1
    for x in range(2, W - 2):            # zigzag over a tile-row edge
        p[min(H - 2, 60 + (x % 3) - 1), x] = 1
    p[H - 6:H - 2, W - 7:W - 2] = 1
    p[H - 4, W - 5] = 0
    return p


@pytest.mark.parametrize("shape", [(64, 64), (120, 161), (91, 149)])
@pytest.mark.parametrize("density", [0.35, 0.5, 0.65])
def test_window_follows_walk_on_noise(shape, density):
    rng = np.random.default_rng(int(density * 100) + shape[0])
    bad, steps, crossings = _window_check((rng.random(shape) < density).astype(np.uint8))
    assert steps > 1000 and crossings > 50
    assert bad == 0


@pytest.mark.parametrize("size,min_crossings", [((1920, 1080), 1000), ((187, 131), 100), ((61, 31), 10), ((31, 29), 1), ((30, 30), 0)])
def test_window_follows_walk_along_tile_and_image_edges(size, min_crossings):
    W, H = size
    bad, steps, crossings = _window_check(_edge_plane(W, H), max_steps=3000)
    assert steps > 20 and crossings >= min_crossings
    assert bad == 0


@pytest.mark.parametrize("ck_step", [1, 3, 4, 7, 256])
def test_trace_segment_writes_its_own_words_at_every_alignment(ck_step):
    rng = np.random.default_rng(ck_step)
    planes = [(rng.random((90, 127)) < 0.55).astype(np.uint8), _edge_plane(187, 131)]
    for plane in planes:
        bad, out = _segment_check(plane, ck_step)
        assert out[0] > 100 and out[1] > 20
        assert all(out[2:6] > 0), out  # every alignment of a segment's first word was met
        assert bad == 0
