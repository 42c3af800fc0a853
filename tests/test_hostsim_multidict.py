"""Detection with several dictionaries on the host (tests/hostsim/multidict_hostsim.cpp) against cv2 4.13's detectMarkersMultiDict over
a seeded sweep.  Ids, marker order and dictionary indices must be identical; corners bit-identical under NONE and within 2e-2 px under
CONTOUR (cv2's sgemm, as tests/test_hostsim_detect.py).  Under SUBPIX a corner may differ by up to 0.05 px, on at most 1 % of the
corners; every other corner within one float32 ulp (2.5e-4).  The looser bound is not an error of the multi-dictionary path: on the
sweep the corners beyond one ulp are those where the single-dictionary host chain already differs from cv2.detectMarkers alone
(cornerSubPix ending on another optimum nearby after a start one ulp apart); test_subpix_outliers_are_single_dictionary checks it.
CPU only."""
import numpy as np
import pytest

import multidict_oracle as mo

CASES = list(mo.sweep_cases(160))
_seen = {"frames": 0, "markers": 0, "dicts": set(), "subpix_corners": 0, "subpix_off": 0}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nmulti-dictionary sweep vs cv2: %d frames, %d markers" % (_seen["frames"], _seen["markers"]))


def assert_corners(name, got, ref, method):
    if method == 0:
        assert np.array_equal(got, ref), name
    elif method == 1:  # cornerSubPix: typically bit-identical, 1 float32 ulp otherwise; now and then another optimum nearby
        err = np.abs(got - ref).reshape(-1, 2).max(axis=1) if len(got) else np.zeros(0)
        assert err.max(initial=0) <= 0.05, (name, err.max())
        _seen["subpix_corners"] += len(err)
        _seen["subpix_off"] += int((err > 2.5e-4).sum())
    else:  # CONTOUR: cv2's sgemm (tests/test_hostsim_detect.py)
        assert np.abs(got - ref).max(initial=0) <= 2e-2, (name, np.abs(got - ref).max(initial=0))


def check(name, bgr, dl, method):
    ids, corners, di = mo.host_multi(bgr, dl, method)
    rids, rcorners, rdi, _ = mo.cv2_multi(bgr, dl, method)
    assert ids.tolist() == rids.tolist(), name
    assert di.tolist() == rdi.tolist(), name
    assert_corners(name, corners, rcorners, method)
    _seen["frames"] += 1
    _seen["markers"] += len(ids)
    _seen["dicts"].update(set(di.tolist()))
    return len(ids)


@pytest.mark.parametrize("k", range(0, len(CASES), 10))
def test_sweep(k):
    for name, bgr, dl, method in CASES[k:k + 10]:
        check(name, bgr, dl, method)


def test_sweep_subpix_rate():
    """cornerSubPix lands on another optimum, a few hundredths of a pixel away, for at most 1 % of the sweep's corners."""
    assert _seen["subpix_corners"] > 500
    assert _seen["subpix_off"] <= 0.01 * _seen["subpix_corners"], (_seen["subpix_off"], _seen["subpix_corners"])


def test_subpix_outliers_are_single_dictionary():
    """Every SUBPIX corner off cv2's multi-dictionary result by more than one ulp is off cv2.detectMarkers for its dictionary alone by
    the same amount: the multi-dictionary path adds no error of its own."""
    n_off = 0
    for name, bgr, dl, method in CASES:
        if method != 1 or name.startswith(("blank", "noise")):
            continue
        ids, corners, di = mo.host_multi(bgr, dl, 1)
        _, rcorners, _, _ = mo.cv2_multi(bgr, dl, 1)
        err = np.abs(corners - rcorners).reshape(len(ids), -1).max(axis=1) if len(ids) else np.zeros(0)
        for d in sorted(set(di[err > 2.5e-4].tolist())):
            _, scorners, _ = mo.cv2_single(bgr, dl[d], 1)
            assert np.array_equal(rcorners[di == d], scorners), (name, d)  # cv2's blocks are its single runs
            n_off += 1
    assert n_off <= 10


def test_sweep_found_markers():
    """The sweep is not vacuous: most rendered frames yield markers of several dictionaries."""
    n_multi = 0
    for name, bgr, dl, method in CASES[:40]:
        if name.startswith(("blank", "noise")):
            continue
        _, _, di = mo.host_multi(bgr, dl, method)
        n_multi += len(set(di.tolist())) > 1
    assert n_multi >= 20, n_multi


def test_concatenation_of_single_runs():
    """Each dictionary's block equals what detectMarkers returns for that dictionary alone (finding 15)."""
    for name, bgr, dl, method in CASES[:21]:
        ids, corners, di = mo.host_multi(bgr, dl, method)
        for d, dict_id in enumerate(dl):
            sids, scorners, _ = mo.cv2_single(bgr, dict_id, method)
            assert ids[di == d].tolist() == sids.tolist(), (name, d)
            assert_corners((name, d), corners[di == d], scorners, method)


def test_nested_family():
    """A marker of the second family inside a white cell of a marker of the first is found by its own dictionary, and so is the
    enclosing marker by the first."""
    import cv2

    dl = mo.DICT_LISTS["sizes_4_6_5"]
    bgr = mo.render_mixed(1280, 720, dl, 7, n_markers=3, nested=True)
    n = check("nested", bgr, dl, 1)
    _, corners, di = mo.host_multi(bgr, dl, 1)
    nested = [(i, j) for i in np.where(di == 0)[0] for j in np.where(di == 1)[0]
              if all(cv2.pointPolygonTest(corners[i].astype(np.float32), (float(x), float(y)), False) > 0 for x, y in corners[j])]
    assert len(nested) == 1, nested
    assert n >= 2
