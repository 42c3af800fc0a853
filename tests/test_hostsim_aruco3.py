"""useAruco3Detection on the host (fiducials_b200/csrc/aruco3.cuh through tests/hostsim/aruco3_hostsim.cpp) against cv2 4.13
(DESIGN.md finding 16): the planes bit for bit against cv2.resize and repeated cv2.pyrDown; a seeded sweep of 160 frames against
cv2.aruco.ArucoDetector(...).detectMarkers with the reference parameters plus the mode (640x480 to 3840x2160, ratios 0 / 0.01 /
0.02 / 0.05, minSide 16 / 32 / 64, DICT_6X6_250, APRILTAG_36h11 and DICT_4X4_50, markers near the minimum side, large, oblique, in
the frame corners and blurred, blank and noise frames); and the rules found by probing, each directly.  Ids and order identical;
corners bit-identical except where cornerSubPix ends a last bit or so away (at most 1 % of corners, each within 0.05 px).  CPU
only."""
import functools

import cv2
import numpy as np
import pytest

import aruco3_oracle as a3

A = a3.A
CASES = list(a3.sweep_cases(160))


@functools.lru_cache(maxsize=None)
def _case(i):
    """(host ids, host corners, cv2 ids, cv2 corners) of sweep case i, computed once per session."""
    name, bgr, d, min_side, ratio = CASES[i]
    return a3.host_detect(bgr, d, min_side, ratio) + a3.cv2_detect(bgr, d, min_side, ratio)


@pytest.mark.parametrize("W,H", [(64, 48), (65, 49), (641, 479), (1280, 720), (1921, 1081), (3840, 2160)])
def test_planes_bit_identical(W, H):
    g = np.random.default_rng(W * H).integers(0, 256, (H, W)).astype(np.uint8)
    g = cv2.GaussianBlur(g, (0, 0), 1.5) if W > 1000 else g  # both textures: noise and smooth
    for min_side in a3.MIN_SIDES:
        for ratio in a3.RATIOS:
            seg, levels, closest = a3.host_planes(g, min_side, ratio)
            rseg, rpyr = a3.cv2_planes(g, min_side, ratio)
            assert seg.shape == rseg.shape and np.array_equal(seg, rseg), (min_side, ratio)
            assert len(levels) == len(rpyr)
            for l, (a, b) in enumerate(zip(levels, rpyr)):
                assert np.array_equal(a, b), (min_side, ratio, l)
            assert closest == a3.geometry(W, H, min_side, ratio)[3]


def test_geometry_of_the_issue_table():
    """Segmentation planes and pyramid depths at the default minSide 32 (cv2's formula in float32)."""
    assert a3.geometry(1920, 1080, 32, 0.02) == (873, 491, 6, 1)
    assert a3.geometry(1920, 1080, 32, 0.05) == (480, 270, 6, 2)
    assert a3.geometry(3840, 2160, 32, 0.02) == (1129, 635, 7, 2)
    assert a3.geometry(3840, 2160, 32, 0.05) == (549, 309, 7, 3)


@pytest.mark.parametrize("k", range(0, len(CASES), 10))
def test_sweep(k):
    for i in range(k, min(k + 10, len(CASES))):
        name, _, _, _, ratio = CASES[i]
        ids, corners, rids, rcorners = _case(i)
        assert ids.tolist() == rids.tolist(), name
        err = np.abs(corners - rcorners).reshape(-1, 2).max(axis=1) if len(ids) else np.zeros(0)
        assert err.max(initial=0) <= 0.05, (name, err.max())
        if ratio == 0:  # no scaling, no cornerSubPix: the corners of the candidate stage
            assert np.array_equal(corners, rcorners), name


def test_sweep_rates():
    """The sweep is not vacuous, and cornerSubPix ends elsewhere for at most 1 % of its corners (measured: 12 of 4 136)."""
    markers = n_corners = off = 0
    for i in range(len(CASES)):
        ids, corners, _, rcorners = _case(i)
        if len(ids) != len(rcorners):
            continue  # test_sweep reports the id mismatch
        err = np.abs(corners - rcorners).reshape(-1, 2).max(axis=1) if len(ids) else np.zeros(0)
        markers += len(ids)
        n_corners += len(err)
        off += int((err > 0).sum())
    print("\naruco3 sweep vs cv2: %d frames, %d markers, %d of %d corners not bit-identical" % (len(CASES), markers, off, n_corners))
    assert markers >= 600
    assert off <= 0.01 * n_corners, (off, n_corners)


def test_refinement_method_is_overridden():
    """With the mode on, NONE, SUBPIX and CONTOUR give the same ids and corners."""
    bgr = a3.render(1920, 1080, A.DICT_6X6_250, 11, 12, side_range=(0.2, 0.8))
    res = [a3.cv2_detect(bgr, A.DICT_6X6_250, 32, 0.02, cornerRefinementMethod=m) for m in (0, 1, 2)]
    hids, hcorners = a3.host_detect(bgr, A.DICT_6X6_250, 32, 0.02)
    assert len(hids) >= 6
    for ids, corners in res:
        assert ids.tolist() == hids.tolist() and np.array_equal(corners, res[0][1])


def test_ratio_zero_gives_unrefined_corners():
    """At ratio 0 the frame is not scaled and no cornerSubPix runs: the corners are those of plain NONE detection."""
    bgr = a3.render(1280, 720, A.DICT_6X6_250, 12, 8, side_range=(0.4, 0.8))
    ids, corners = a3.host_detect(bgr, A.DICT_6X6_250, 32, 0.0)
    det = A.ArucoDetector(A.getPredefinedDictionary(A.DICT_6X6_250), a3.ao.reference_detector_params(cornerRefinementMethod=0))
    rcorners, rids, _ = det.detectMarkers(bgr)
    assert len(ids) >= 4 and ids.tolist() == rids.reshape(-1).tolist()
    assert np.array_equal(corners, np.array(rcorners, np.float32).reshape(-1, 4, 2))


def test_perimeter_rule():
    """minMarkerPerimeterRate gives way to a minimum contour length of 4 * minSide: a 40 px marker in a 1080p frame is below the
    reference's rate (0.1 * 1920 = 192 points) and found with the mode; a marker whose sides in the segmentation plane fall well
    below minSide is dropped."""
    g = np.full((1080, 1920), 200, np.uint8)
    m = a3._marker(A.DICT_6X6_250, 7, 40)
    g[500:540, 900:940] = m
    big = a3._marker(A.DICT_6X6_250, 9, 300)
    g[100:400, 100:400] = big
    bgr = np.ascontiguousarray(cv2.cvtColor(g, cv2.COLOR_GRAY2BGR))
    plain, _ = a3.ao.detect(bgr, A.DICT_6X6_250)
    assert sorted(plain.tolist()) == [9]
    ids, _ = a3.host_detect(bgr, A.DICT_6X6_250, 16, 0.0)
    assert sorted(ids.tolist()) == [7, 9] and ids.tolist() == a3.cv2_detect(bgr, A.DICT_6X6_250, 16, 0.0)[0].tolist()
    # at ratio 0.05 the segmentation plane is 273 wide: the 40 px marker is ~6 px there, far below minSide 16
    ids, _ = a3.host_detect(bgr, A.DICT_6X6_250, 16, 0.05)
    assert ids.tolist() == [9] and a3.cv2_detect(bgr, A.DICT_6X6_250, 16, 0.05)[0].tolist() == [9]


def test_level_choice():
    """The level whose scaled contour length exceeds 4 * minSide by the least, level 0 when none does (1080p, ratio 0.02: the
    segmentation plane is 873 wide, levels 1920, 960, 480, 240, 120, 60 wide)."""
    sw = 873
    widths = [1920, 960, 480, 240, 120, 60]
    for n in [10, 128, 129, 200, 300, 600, 1000, 3000]:
        best, dist = 0, np.float32(np.inf)
        for i, w in enumerate(widths):
            nd = np.float32(n) * (np.float32(w) / np.float32(sw)) - np.float32(128)
            if nd < dist and nd > 0:
                best, dist = i, nd
        assert a3.host_level_for(1920, 1080, 32, 0.02, n) == best, n
    assert a3.host_level_for(1920, 1080, 32, 0.02, 10) == 0


def test_window_rule():
    """cornerSubPix runs with window 5 on levels whose larger side is above 1080 and 3 otherwise: on a 4K frame at ratio 0.05 the
    corners pass through levels 2 (960), 1 (1920) and 0 (3840); with that rule the host chain matches cv2 bit for bit here."""
    bgr = a3.render(3840, 2160, A.DICT_6X6_250, 13, 12, side_range=(0.3, 0.7))
    assert a3.geometry(3840, 2160, 32, 0.05)[3] == 3
    ids, corners = a3.host_detect(bgr, A.DICT_6X6_250, 32, 0.05)
    rids, rcorners = a3.cv2_detect(bgr, A.DICT_6X6_250, 32, 0.05)
    assert len(ids) >= 6 and ids.tolist() == rids.tolist()
    assert np.array_equal(corners, rcorners)
