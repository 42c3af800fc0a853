"""The composition that boards bound to dictionary families follow (DESIGN.md finding 19), pinned against cv2 on seeded frames with
colliding raw ids: each family's markers are one contiguous run of detectMarkersMultiDict's list, equal to detectMarkers with that
family alone; the board stages on that run equal the single-family runs; the unfiltered list takes the other family's markers; and
the host build of board_pnp.cuh's matching, fed the run as the device feeds it, agrees with Board.matchImagePoints.  CPU only."""
import numpy as np
import pytest

import board_oracle as bo
import charuco_oracle as co
import multidict_boards_cases as mc
import multidict_oracle as mo
from fiducials_b200 import synth

A = mc.A
K, D = synth.camera_for(mc.W, mc.H)
GRIDS = [A.DICT_4X4_50, A.DICT_5X5_1000]
MIXED = [A.DICT_6X6_250, A.DICT_APRILTAG_36h11, A.DICT_4X4_50]


def _runs_contiguous(di):
    return all(a <= b for a, b in zip(di[:-1], di[1:]))


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("method", [0, 1])
def test_family_run_is_the_single_family_detection(seed, method):
    for bgr, dicts in ((mc.render_grids(seed), GRIDS), (mc.render_mixed_boards(seed), MIXED), (mc.render_grids(seed, (A.DICT_4X4_50,) * 2), [A.DICT_4X4_50] * 2)):
        ids, corners, di = mc.cv2_multi(bgr, dicts, method)
        assert _runs_contiguous(di.tolist())
        for k, d in enumerate(dicts):
            fi, fc = mc.family(ids, corners, di, k)
            si, sc = mc.cv2_single(bgr, d, method)
            assert fi.tolist() == si.tolist() and np.array_equal(fc, sc), (seed, k)


@pytest.mark.parametrize("seed", [0, 1])
def test_board_pose_on_the_run_equals_the_single_family_pose(seed):
    bgr = mc.render_grids(seed)
    ids, corners, di = mc.cv2_multi(bgr, GRIDS)
    board = mc.grid()
    for k, d in enumerate(GRIDS):
        si, sc = mc.cv2_single(bgr, d)
        got = bo.board_pose(board, *mc.family(ids, corners, di, k), K, D)
        ref = bo.board_pose(board, si, sc, K, D)
        assert got["status"] == 1 and got["n_markers"] == 4
        bo.assert_matches(got, ref, "family %d" % k, tol=0.0)


@pytest.mark.parametrize("seed", [0, 1])
def test_unfiltered_list_takes_the_other_familys_markers(seed):
    """Why a board needs its family: Board.matchImagePoints and CharucoDetector.detectBoard on the whole multi-dictionary list take
    the markers of every family whose raw ids are on the board."""
    bgr = mc.render_grids(seed)
    ids, corners, di = mc.cv2_multi(bgr, GRIDS)
    board = mc.grid()
    obj_all, _ = bo.match(board, ids, corners)
    obj_fam, _ = bo.match(board, *mc.family(ids, corners, di, 0))
    assert len(obj_all) == 2 * len(obj_fam) == 32
    assert bo.board_pose(board, ids, corners, K, D)["n_markers"] == 8
    bgr = mc.render_mixed_boards(seed)
    gray = cv2_gray(bgr)
    ids, corners, di = mc.cv2_multi(bgr, MIXED)
    cb = mc.cv_charuco(mc.charuco(), MIXED[0])
    fi, fc = mc.family(ids, corners, di, 0)
    markers = A.Board(cb.getObjPoints(), cb.getDictionary(), cb.getIds())  # the markers detectBoard's approximate pose matches
    obj_all, _ = markers.matchImagePoints(list(corners.reshape(-1, 1, 4, 2)), ids.reshape(-1, 1))
    obj_fam, _ = markers.matchImagePoints(list(fc.reshape(-1, 1, 4, 2)), fi.reshape(-1, 1))
    assert len(obj_fam) == 40 and len(obj_all) == 96  # the AprilTags 0..9 and the 4x4 markers 0..3 collide with the board's ids
    all_ids, all_xy = co.detect(cb, gray, ids, corners, K, D)
    fam_ids, fam_xy = co.detect(cb, gray, fi, fc, K, D)
    assert len(fam_ids) == 12
    assert not (np.array_equal(all_ids, fam_ids) and np.array_equal(all_xy, fam_xy))


def cv2_gray(bgr):
    import cv2

    return cv2.cvtColor(bgr, cv2.COLOR_BGR2GRAY)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_host_matching_on_the_run_agrees_with_cv2(seed):
    """The host chain's multi-dictionary list (tests/hostsim/multidict_hostsim.cpp) keeps each family in one run; board_pnp.cuh's
    matching on that run (host build, tests/hostsim/board_hostsim.cpp) equals matchImagePoints on corners[di == k]."""
    import test_hostsim_board as hb

    for bgr, dicts, board in ((mc.render_grids(seed), GRIDS, mc.grid()), (mc.render_mixed_boards(seed), MIXED, mc.grid())):
        hids, hcorners, hdi = mo.host_multi(bgr, dicts, 1)
        rids, _, rdi, _ = mo.cv2_multi(bgr, dicts, 1)
        assert hids.tolist() == rids.tolist() and hdi.tolist() == rdi.tolist()
        assert _runs_contiguous(hdi.tolist())
        for k in range(len(dicts)):
            lo, hi = int(np.searchsorted(hdi, k, "left")), int(np.searchsorted(hdi, k, "right"))
            obj, img = hb.hs_match(board, hids[lo:hi], hcorners[lo:hi])
            robj, rimg = bo.match(board, *mc.family(hids, hcorners, hdi, k))
            assert np.array_equal(obj, robj) and np.array_equal(img, rimg), (seed, k)
