"""detectInvertedMarker (DESIGN.md finding 18) on the CPU: the host chain of tests/hostsim/inverted_hostsim.cpp, which runs
identify.cuh's two-polarity variant (identify_candidate<CONF, true>) and quad_group.cuh's smallest-first grouping
(group_candidates<true>), against cv2 4.13 with the flag; and probes that pin findings A and B on their own."""
import cv2
import numpy as np
import pytest

import inverted_oracle as io
from oracle import aruco_oracle as ao

A = io.A
# corners against cv2 under SUBPIX and CONTOUR: the single-dictionary tolerance of the host chain (cornerSubPix and the line fit
# run in float with another operation order than cv2's SIMD code)
TOL = {"none": 0.0, "subpix": 0.05, "contour": 0.05}


@pytest.mark.parametrize("case", list(io.sweep_cases(120)), ids=lambda c: c[0])
def test_sweep_matches_cv2(case):
    """Ids and their order identical on every frame, corners bit-identical under NONE and within the tolerance otherwise."""
    name, g, dict_id, kw = case
    ci, cc, _ = io.cv2_detect(g, dict_id, **kw)
    hi, hc, _, _ = io.host_detect(g, dict_id, **kw)
    assert ci.tolist() == hi.tolist()
    assert np.abs(cc - hc).max(initial=0) <= TOL[kw["method"]]


def test_sweep_covers_both_polarities_and_the_flag_off():
    """The sweep finds white and black markers, and with the flag off the host chain is cv2's plain detectMarkers."""
    n_white = n_black = 0
    for name, g, dict_id, kw in list(io.sweep_cases(120))[::4]:
        _, _, _, pol = io.host_detect(g, dict_id, **kw)
        n_white += int(pol.sum())
        n_black += int((pol == 0).sum())
        ci, cc, _ = io.cv2_detect(g, dict_id, inverted=False, **kw)
        hi, hc, _, hp = io.host_detect(g, dict_id, inverted=False, **kw)
        assert ci.tolist() == hi.tolist() and not hp.any(), name
        assert np.abs(cc - hc).max(initial=0) <= TOL[kw["method"]], name
    assert n_white > 30 and n_black > 30, (n_white, n_black)


def test_blank_frames():
    for name, g in io.blank_frames():
        assert io.cv2_detect(g, A.DICT_6X6_250)[0].tolist() == io.host_detect(g, A.DICT_6X6_250)[0].tolist() == [], name


def _pow2(win):
    return win & (win - 1) == 0


def test_confidence_matches_cv2():
    """As finding 17: bit-identical where the window area is a power of two, within 1e-6 otherwise; white markers score against
    the polarity that was chosen."""
    n = n_white = 0
    for name, g, dict_id, kw in list(io.sweep_cases(120))[::3]:
        for ppc, margin in ((kw["ppc"], 0.13), (4, 0.0)):
            k = dict(kw, ppc=ppc, margin=margin)
            ci, _, cf = io.cv2_detect_conf(g, dict_id, **k)
            hi, _, hf, hp = io.host_detect(g, dict_id, **k)
            assert ci.tolist() == hi.tolist(), name
            win = ppc - 2 * int(margin * ppc)
            if _pow2(win * win):
                assert np.array_equal(cf, hf), (name, cf, hf)
            else:
                assert np.abs(cf.astype(np.float64) - hf).max(initial=0) <= 1e-6, name
            n += len(hi)
            n_white += int(hp.sum())
    assert n > 200 and n_white > 60
    g = io.lone_marker(white=True)
    assert io.cv2_detect_conf(g, A.DICT_6X6_250, ppc=4, margin=0.0)[2].tolist() == io.host_detect(g, A.DICT_6X6_250, ppc=4, margin=0.0)[2].tolist()


# ---- finding A: two polarities per candidate ------------------------------------------------------------------------------------


def _quad(g, dict_id=A.DICT_6X6_250):
    """The corners cv2 returns with NONE for the only marker of g (the candidate identification reads)."""
    ids, corners, _ = io.cv2_detect(g, dict_id, method="none")
    assert len(ids) == 1
    return corners[0]


def test_white_marker_is_read_inverted():
    g = io.lone_marker(px=15, white=True)
    assert io.cv2_detect(g, A.DICT_6X6_250, inverted=False)[0].tolist() == []
    q = _quad(g)
    i, _, pol, _ = io.host_identify(g, q, A.DICT_6X6_250)
    assert (i, pol) == (7, 1)
    assert io.host_identify(g, q, A.DICT_6X6_250, inverted=False)[0] == -1


@pytest.mark.parametrize("bb", [1, 2])
def test_tie_keeps_the_cells_as_read(bb):
    """Border errors equal in both polarities (half the border ring white): the cells stay as read -- the marker whose inner cells
    are the normal reading decodes, the inverted reading's id does not."""
    d = A.getPredefinedDictionary(A.DICT_4X4_50)
    cells = 4 + 2 * bb
    px = 12
    bits = np.zeros((cells, cells), np.uint8)
    bits[bb:-bb, bb:-bb] = d.getBitsFromByteList(d.bytesList[3:4], 4)
    ring = [(y, x) for y in range(cells) for x in range(cells) if y < bb or y >= cells - bb or x < bb or x >= cells - bb]
    for y, x in ring[: len(ring) // 2]:
        bits[y, x] = 1
    m = np.kron(bits * 255, np.ones((px, px), np.uint8)).astype(np.uint8)
    g = np.full((cells * px + 100, cells * px + 100), 128, np.uint8)
    g[50:50 + cells * px, 50:50 + cells * px] = m
    q = np.float32([[50, 50], [50 + cells * px - 1, 50], [50 + cells * px - 1, 50 + cells * px - 1], [50, 50 + cells * px - 1]])
    kw = dict(method="none", border_bits=bb, ecr=0.0, border_rate=2.0)
    i, rot, pol, _ = io.host_identify(g, q, A.DICT_4X4_50, **kw)
    assert (i, rot, pol) == (3, 0, 0)
    # the same cells inverted decode only as a white marker: strictly fewer errors inverted
    i, rot, pol, _ = io.host_identify(255 - g, q, A.DICT_4X4_50, **kw)
    assert (i, pol) == (-1, 0)  # still a tie: read as is, and the inverted word is no marker


def test_probe_numbers_of_the_issue():
    """1280 x 720 frames of 12 DICT_6X6_250 markers, reference parameters (SUBPIX): inverted, cv2 finds none without the flag and
    all 12 with it, within 0.006 px of the normal-polarity detection of the same frame."""
    from fiducials_b200 import synth

    for seed in range(3):
        img = synth.make_frame(1280, 720, 12, A.DICT_6X6_250, seed=seed)
        g = ao.gray(img[0] if isinstance(img, tuple) else img)
        assert len(io.cv2_detect(255 - g, A.DICT_6X6_250, inverted=False)[0]) == 0
        ni, nc, _ = io.cv2_detect(g, A.DICT_6X6_250, inverted=False)
        wi, wc, _ = io.cv2_detect(255 - g, A.DICT_6X6_250)
        hi, hc, _, hp = io.host_detect(255 - g, A.DICT_6X6_250)
        assert len(wi) == 12 and hi.tolist() == wi.tolist() and hp.all()
        ref = {int(i): c for i, c in zip(ni, nc)}
        assert max(np.abs(c - ref[int(i)]).max() for i, c in zip(wi, wc)) < 0.006


# ---- finding B: the group keeps its smallest member -----------------------------------------------------------------------------


def test_lone_marker_keeps_the_inner_outline():
    """A lone 120 px marker at (50, 50): the flag moves its first corner (50, 50) inward to the smallest outline of its group,
    (56, 57) -- bit for bit in the host chain."""
    g = io.lone_marker(px=15)
    for inv, first in ((False, (50.0, 50.0)), (True, (56.0, 57.0))):
        ci, cc, _ = io.cv2_detect(g, A.DICT_6X6_250, inv, method="none")
        hi, hc, _, _ = io.host_detect(g, A.DICT_6X6_250, inv, method="none")
        assert ci.tolist() == hi.tolist() == [7] and np.array_equal(cc, hc)
        assert tuple(float(v) for v in cc[0, 0]) == first


def test_black_markers_change_order_and_corners_with_the_flag():
    """On the issue's frames the flag reorders black markers and moves their corners 6-10 px inward; most SUBPIX corners stay
    integers (cornerSubPix has no gradient inside the black border).  The host chain reproduces all of it."""
    from fiducials_b200 import synth

    n_int = n = 0
    reordered = False
    for seed in range(3):
        img = synth.make_frame(1280, 720, 12, A.DICT_6X6_250, seed=seed)
        g = ao.gray(img[0] if isinstance(img, tuple) else img)
        ai, ac, _ = io.cv2_detect(g, A.DICT_6X6_250, inverted=False)
        bi, bc, _ = io.cv2_detect(g, A.DICT_6X6_250)
        hi, hc, _, hp = io.host_detect(g, A.DICT_6X6_250)
        assert hi.tolist() == bi.tolist() and not hp.any()
        assert np.abs(bc - hc).max() <= TOL["subpix"]
        reordered |= ai.tolist() != bi.tolist()
        ref = {int(i): c for i, c in zip(ai, ac)}
        shift = [np.abs(c - ref[int(i)]).max() for i, c in zip(bi, bc) if int(i) in ref]
        assert min(shift) > 5 and max(shift) < 11
        n_int += sum(int(np.array_equal(c, np.round(c))) for c in bc)
        n += len(bi)
    assert reordered and n_int > n // 2


@pytest.mark.parametrize("kind", ["nested", "oblique", "blur"])
def test_group_rule_on_nested_oblique_blurred_and_multiscale(kind):
    """The smallest-first rule, pinned on frames where groups are deep: a marker nested in another's quiet zone, strong
    perspective, blur, and three frame sizes -- ids, order and NONE corners bit-identical with cv2."""
    n = 0
    for s, (W, H) in enumerate(io.SIZES):
        g = io.render(1200 + s, A.DICT_6X6_250, 1, kind, "mixed", W, H, n_markers=6)
        ci, cc, _ = io.cv2_detect(g, A.DICT_6X6_250, method="none")
        hi, hc, _, _ = io.host_detect(g, A.DICT_6X6_250, method="none")
        assert ci.tolist() == hi.tolist() and np.array_equal(cc, hc), (W, H)
        n += len(ci)
    assert n >= 8
