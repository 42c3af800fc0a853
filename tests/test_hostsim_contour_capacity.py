"""The contour-stage cases of tests/contour_cases.py do what they were built for, counted on the CPU: the fine textures overflow the
start-crack queue (or fit it), the segments pass the chain capacity, the lines the point capacity, the walk-round and length-filter
cases have the contours they are named for.  The start-crack bound the replay rests on (at most 15 left and 15 right cracks per 30-pixel
tile row and plane) holds on random planes and is reached by the 1-pixel checkerboard.  The host build of the device's start rules
and border walk finds cv2's contours on the texture planes.  CPU only."""
import ctypes as C

import cv2
import numpy as np
import pytest

import contour_cases as cc
import hostsim_util as hs
from oracle import aruco_oracle as ao

MAX_CHAINS = 65536
# the cases whose in-range contours are counted here (the others' counts cost cv2 minutes: millions of contours per plane)
COUNTED = [n for n in cc.CASES if not n.endswith("_uhd") and not (n.endswith("full_fhd") and cc.CASES[n]["texture"] in ("checker1", "dither1"))]


def _planes(name):
    return ao.threshold_planes(ao.gray(cc.render(name)[0]))


@pytest.mark.parametrize("name", sorted(cc.CASES))
def test_start_queue_band(name):
    """Start cracks of the frame against the queue of a one-frame chunk, per side."""
    c = cc.CASES[name]
    W, H = c["W"], c["H"]
    n = cc.start_counts(_planes(name)).sum(0)
    over = bool((n > cc.start_queue_cap(W, H)).any())
    assert over == (cc.expect(name)["queue"] == "over"), (name, n / (W * H))
    assert (n <= 13 * ((W + 1) // 2) * H).all()  # the bound: one crack per two pixels of a row, plane and side


@pytest.mark.parametrize("name", sorted(COUNTED))
def test_contour_capacity_band(name):
    c = cc.CASES[name]
    W, H = c["W"], c["H"]
    chains, points = cc.in_range_counts(_planes(name), W, H)
    e = cc.expect(name)
    hw, hh = cc.handle(name)
    assert (chains > MAX_CHAINS) == (e["chains"] == "over"), (name, chains)
    assert (points > 4 * hw * hh + 65536) == (e["points"] == "over"), (name, points)


def test_chain_capacity_needs_a_frame_smaller_than_its_handle():
    """65536 in-range contours of min_len points each exceed the point capacity of a handle the frame fills unless its shorter side
    is 1639 pixels or more; the segments frame is 1280 x 720 in a 3840 x 2160 handle."""
    for W, H in ((640, 480), (1280, 720), (1920, 1080), (1920, 1200)):
        assert MAX_CHAINS * cc.min_len(W, H) > 4 * W * H + 65536
    W, H = 1280, 720
    hw, hh = cc.handle("segments_hd_in_uhd")
    assert MAX_CHAINS * cc.min_len(W, H) < 4 * hw * hh + 65536


def test_walk_round_cases():
    """spiral: a contour longer than every bounded round's budget (8 + 64 + 512 steps) and in range; serpentine: one past max_len."""
    for name, lo, hi in (("spiral_fhd", 585, cc.max_len(1920, 1080)), ("serpentine_fhd", cc.max_len(1920, 1080) + 1, 1 << 30)):
        n = cc.contour_lengths(_planes(name)[6])
        assert ((n >= lo) & (n <= hi)).any(), name


def test_length_filter_cases():
    """Contours of exactly min_len - 1, min_len and max_len, max_len + 1 points on every plane; the min_len - 1 and min_len ones are
    convex 4-gons, so cv2's candidates have the min_len quads and none of min_len - 1 points."""
    lo, hi = cc.min_len(640, 480), cc.max_len(640, 480)
    assert lo == 64 and hi == 2560  # the reference's perimeter rates 0.1 and 4.0
    for name, lens in (("length_min_vga", (lo - 1, lo)), ("length_max_vga", (hi, hi + 1))):
        for p in _planes(name):
            n = set(cc.contour_lengths(p).tolist())
            assert set(lens) <= n, (name, lens)
    for n in (lo - 1, lo):
        cs, _ = cv2.findContours(cc._quad_mask(n).astype(np.uint8), cv2.RETR_EXTERNAL, cv2.CHAIN_APPROX_NONE)
        assert len(cs[0]) == n and len(cv2.approxPolyDP(cs[0], 0.01 * n, True)) == 4
    raw = {n for _, _, n in ao.quad_candidates(ao.gray(cc.render("length_min_vga")[0]))}
    assert lo in raw and lo - 1 not in raw


def test_seam_cases_cross_the_tile_seams():
    """The seam frames: one pixel either side of a tile multiple, and the markers' outer edges at x, y = 0, 1, 29 (mod 30)."""
    sizes = {(c["W"] % cc.HALO_T, c["H"] % cc.HALO_T) for n, c in cc.CASES.items() if c["kind"] == "seams"}
    assert {(29, 29), (0, 0), (1, 1)} <= sizes
    bgr, ids = cc.render("seams_600x450")
    rids, rc = ao.detect(bgr, cc.DICT)
    assert set(rids.tolist()) == ids
    assert {int(round(float(rc[:, :, 0].min(axis=1)[k]))) % cc.HALO_T for k in range(len(rids))} == {0, 1, 29}


@pytest.mark.parametrize("seed", range(4))
def test_start_bound_on_random_planes(seed):
    """At most 15 left and 15 right start cracks per tile row of 30 interior pixels and plane -- the host build of halo_row_starts
    over every tile, against the numpy restatement -- and the 1-pixel checkerboard reaches it."""
    lib = hs.load()
    rng = np.random.default_rng(seed)
    H, W = 97, 151
    for density in (0.3, 0.5, 0.7):
        plane = (rng.random((H, W)) < density).astype(np.uint8)
        left, right = cc.row_starts(plane)
        for m in (left, right):
            per_tile_row = np.add.reduceat(m.astype(np.int64), np.arange(0, W, cc.HALO_T), axis=1)
            assert per_tile_row.max() <= cc.HALO_T // 2
        out = np.zeros(2, np.int64)
        zeros = np.zeros(1 << 15, np.uint8)
        lib.hs_prune_gain(plane.ctypes.data_as(C.c_void_p), W, H, 5, zeros.ctypes.data_as(C.c_void_p), zeros.ctypes.data_as(C.c_void_p),
                          out.ctypes.data_as(C.c_void_p))
        assert out[0] == left.sum() + right.sum()
    y, x = np.mgrid[0:H, 0:W]
    left, right = cc.row_starts(((x + y) & 1).astype(np.uint8))
    inner = left[1:-1, cc.HALO_T : W - W % cc.HALO_T]  # tiles away from the frame's left border
    assert (np.add.reduceat(inner.astype(np.int64), np.arange(0, inner.shape[1], cc.HALO_T), axis=1) == cc.HALO_T // 2).all()


@pytest.mark.parametrize("name", ["checker1_half_vga", "dither1_full_vga", "checker2_full_vga", "noise_half_vga"])
def test_find_contours_on_texture_planes(name):
    """The host build of the start rules and the walk (the GPU's rounds and segments) gives cv2's contours on the texture planes."""
    planes = _planes(name)
    for s in (0, 6, 12):
        ours, nstarts = hs.find_contours(planes[s], mode=1)
        ref = ao.find_contours(planes[s])
        assert len(ours) == len(ref) and all(np.array_equal(a, b) for a, b in zip(ours, ref)), (name, s)
        left, right = cc.row_starts(planes[s])
        assert nstarts == left.sum() + right.sum(), (name, s)
