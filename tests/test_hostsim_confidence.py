"""Detection with confidence (DESIGN.md finding 17) on the CPU: the host chain of tests/hostsim/confidence_hostsim.cpp, which runs
identify.cuh's confidence variant (identify_candidate<true>, marker_confidence), against cv2 4.13's detectMarkersWithConfidence."""
import cv2
import numpy as np
import pytest

import confidence_oracle as co

A = cv2.aruco


@pytest.mark.parametrize("case", co.fixed_cases(), ids=lambda c: c[0])
def test_fixed_cases_match_cv2(case):
    """The probed values: cv2 with its default parameters, cv2 with the reference parameters and the host chain all give them."""
    name, g, dict_id, kw, expected = case
    p = A.DetectorParameters()
    p.perspectiveRemovePixelPerCell = kw["ppc"]
    p.markerBorderBits = kw.get("border_bits", 1)
    _, ids, conf, _ = A.ArucoDetector(A.getPredefinedDictionary(dict_id), p).detectMarkersWithConfidence(g)
    assert ids is not None and len(ids) == 1
    assert np.float32(conf.reshape(-1)[0]) == np.float32(expected)
    ci, _, cf = co.cv2_detect(g, dict_id, **kw)
    hi, _, hf = co.host_detect(g, dict_id, **kw)
    assert ci.tolist() == hi.tolist() and len(hi) == 1
    assert cf[0] == np.float32(expected) and hf[0] == np.float32(expected)


def _pow2(win):
    return win & (win - 1) == 0


def test_seeded_sweep_matches_cv2():
    """Ids identical; confidence identical in float32 where the window area win^2 is a power of two (every share is then a
    dyadic fraction and any summation order is exact) and within 1e-6 otherwise (cv2's summation order is not pinned)."""
    n_markers = n_below_one = 0
    for name, g, dict_id, kw in co.sweep_cases():
        ci, cc, cf = co.cv2_detect(g, dict_id, **kw)
        hi, hc, hf = co.host_detect(g, dict_id, **kw)
        assert ci.tolist() == hi.tolist(), name
        if kw["method"] == "none":
            assert np.array_equal(cc, hc), name
        win = kw["ppc"] - 2 * int(kw["margin"] * kw["ppc"])
        if _pow2(win * win):
            assert np.array_equal(cf, hf), (name, cf, hf)
        else:
            assert np.abs(cf.astype(np.float64) - hf).max(initial=0) <= 1e-6, (name, cf, hf)
        n_markers += len(ci)
        n_below_one += int((cf < 1).sum())
    assert n_markers > 500 and n_below_one > 200, (n_markers, n_below_one)


def test_error_corrected_cells_cost_their_whole_share():
    """A fully inverted inner cell that error correction fixed counts as wrong: the confidence is the dictionary word's, not the
    extracted bits'."""
    g, x0, y0, _ = co.marker_frame(px=20)
    co.paint(g, x0, y0, 20, 2, 2)
    co.paint(g, x0, y0, 20, 4, 5)
    co.paint(g, x0, y0, 20, 6, 3)
    ids, _, conf = co.host_detect(g, A.DICT_6X6_250, ppc=4)
    assert ids.tolist() == [7]
    assert conf[0] == np.float32(1 - 3 / 64)
    assert co.cv2_detect(g, A.DICT_6X6_250, ppc=4)[2][0] == conf[0]


@pytest.mark.parametrize("white", [False, True])
def test_min_otsu_stddev_rule(white):
    """Where the canonical image's inner region has a standard deviation below minOtsuStdDev no threshold is computed: every cell
    counts as all white (mean above 127) or all black, as its bit.  A black or a white square decodes there with a high
    errorCorrectionRate (and, for white, a permissive border rate), and its confidence is that of the all-black or all-white
    grid against the word."""
    g = np.full((400, 400), 0 if white else 255, np.uint8)
    g[100:220, 100:220] = 240 if white else 0
    p = A.DetectorParameters()  # cv2's defaults: 4 pixels per cell, no refinement
    p.errorCorrectionRate = 4.0
    p.maxErroneousBitsInBorderRate = 2.0
    _, ids, conf, _ = A.ArucoDetector(A.getPredefinedDictionary(A.DICT_4X4_50), p).detectMarkersWithConfidence(g)
    assert ids is not None and len(ids) == 1
    d = A.getPredefinedDictionary(A.DICT_4X4_50)
    word = d.getBitsFromByteList(d.bytesList[int(ids[0, 0]):int(ids[0, 0]) + 1], 4)
    ones = int(word.sum())
    wrong = 20 + 16 - ones if white else ones  # white: every border cell and the word's zeros; black: the word's ones
    expected = np.float32(1) - np.float32(wrong) / np.float32(36)
    assert np.float32(conf.reshape(-1)[0]) == expected
    # the host identification of the same quad: the candidate cv2 decoded, from cv2's unrefined corners
    corners, _, _, _ = A.ArucoDetector(A.getPredefinedDictionary(A.DICT_4X4_50), p).detectMarkersWithConfidence(g)
    q = np.array(corners[0], np.float32).reshape(4, 2)
    hid, _, hconf = co.host_identify(g, q, A.DICT_4X4_50, method="none", ppc=4, ecr=4.0, border_rate=2.0)
    assert hid == int(ids[0, 0])
    assert np.float32(hconf) == np.float32(expected)
