"""ChArUco corners and pose on the device (fid_set_charuco_boards, fid_detect_charuco, fid_last_charuco) against cv2's
CharucoDetector.detectBoard + solvePnP and the host build of the same arithmetic, and the default outputs with ChArUco boards set
and without."""
import ctypes as C

import cv2
import numpy as np
import pytest

from fiducials_b200 import _lib, synth
from fiducials_b200.board import charuco_board, grid_board
from fiducials_b200.node import MAXM, Detector, default_params
import charuco_oracle as co
from test_hostsim_charuco import check, hs_detect

pytestmark = pytest.mark.gpu

W, H = 1280, 720
K_R, _ = synth.camera_for(W, H)
D_ZERO = np.zeros(5)
FLEN = 0.14


def _frames(n, seed, boards):
    """n BGR frames, each with the given ChArUco boards side by side; every 3rd frame without any board."""
    rng = np.random.default_rng(seed)
    out = []
    for f in range(n):
        g = np.full((H, W), 128, np.uint8)
        if f % 3 != 2:
            for bi, b in enumerate(boards):
                cvb = co.cv_board(b.size, b.square_length, b.marker_length, b.ids, b.legacy)
                u = W * (bi + 0.5) / len(boards)
                R, t = co.board_pose_in_view(cvb, rng, K_R, W // len(boards), H, kind="near", centre=(u, H / 2 + rng.uniform(-40, 40)))
                co.render(g, cvb, R, t, K_R)
        out.append(cv2.cvtColor(co.blur_noise(g, rng), cv2.COLOR_GRAY2BGR))
    return np.ascontiguousarray(np.stack(out))


BOARD_A = charuco_board((5, 7), 0.03, 0.022)
BOARD_B = charuco_board((4, 4), 0.035, 0.026, ids=list(range(100, 108)))


def _records(det, frame, ids, corners, K):
    return det.charuco(frame, ids, corners, K, None if K is None else D_ZERO)


@pytest.mark.parametrize("camera", [False, True])
def test_detect_charuco_matches_host_and_cv2(camera):
    frames = _frames(6, 1, [BOARD_A, BOARD_B])
    det = Detector(default_params(dictionary=co.DICT_ID), 0, W, H, 2)
    det.set_charuco_boards([BOARD_A, BOARD_B])
    K = K_R if camera else None
    n_corners = 0
    for f, frame in enumerate(frames):
        counts, ids, corners, _ = det.detect_pose_batch(frame[None], K_R, D_ZERO, FLEN)
        n = int(counts[0])
        ids, corners = ids[0, :n], corners.reshape(1, MAXM, 8)[0, :n]
        gray = cv2.cvtColor(frame, cv2.COLOR_BGR2GRAY)
        for bi, (r, cid, cxy) in enumerate(_records(det, frame, ids, corners, K)):
            b = (BOARD_A, BOARD_B)[bi]
            assert r.board == bi and r.n_corners == len(cid)
            hi, hx, hp = hs_detect(b, gray, ids, corners, K, D_ZERO)
            assert np.array_equal(cid, hi) and np.array_equal(cxy, hx), (f, bi)  # the host build, bit for bit
            assert r.status == hp["status"]
            if r.status == 1:
                # the device's double sin / cos / exp differ from the host C library's in the last bit for some arguments and the LM
                # trajectory carries that rounding (measured up to 5e-10 on an H100)
                assert np.abs(np.array(list(r.tvec)) - hp["tvec"]).max() <= 1e-8 and np.abs(np.array(list(r.rvec)) - hp["rvec"]).max() <= 1e-8
            if n:
                check(b, gray, ids, corners, K, D_ZERO, "frame %d board %d" % (f, bi))
            n_corners += len(cid)
    assert n_corners >= 80
    det.close()


def test_batches_match_single_frame_calls_and_defaults_unchanged():
    frames = _frames(9, 2, [BOARD_A, BOARD_B])
    det = Detector(default_params(dictionary=co.DICT_ID), 0, W, H, 4)  # 3 chunks per 9-frame batch
    det.set_pose_hypotheses(True)
    det.set_boards([grid_board((2, 2), 0.03, 0.01, [40, 41, 42, 43])])
    res = []
    for boards in ([], [BOARD_A, BOARD_B], []):
        det.set_charuco_boards(boards)
        det.submit_batch(frames, K_R, D_ZERO, FLEN)
        counts, ids, corners, tfs = det.collect_batch()
        res.append((counts.tobytes(), ids.tobytes(), corners.tobytes(), bytes(tfs), bytes(det.last_pose_hypotheses()),
                    [bytes(r) for fr in det.last_board_poses() for r in fr]))
        if boards:
            ch = det.last_charuco()
            assert len(ch) == len(frames)
            for f in range(len(frames)):
                n = int(counts[f])
                single = det.charuco(frames[f], ids[f, :n], corners.reshape(len(frames), MAXM, 8)[f, :n], K_R, D_ZERO)
                for (r1, i1, x1), (r2, i2, x2) in zip(ch[f], single):
                    assert bytes(r1) == bytes(r2) and np.array_equal(i1, i2) and np.array_equal(x1, x2)
                if f % 3 == 2:
                    assert all(r.n_corners == 0 and r.status == 0 for r, _, _ in ch[f])
    assert res[0] == res[1] == res[2]
    # a batch without a camera: corners, no pose
    det.set_charuco_boards([BOARD_A])
    det.submit_batch(frames)
    det.collect_batch()
    ch = det.last_charuco()
    assert sum(r.n_corners for fr in ch for r, _, _ in fr) > 0 and all(r.status == 0 for fr in ch for r, _, _ in fr)
    det.close()


def test_errors():
    det = Detector(default_params(dictionary=co.DICT_ID), 0, 640, 480, 2)
    lib = det.lib
    frame = np.zeros((480, 640, 3), np.uint8)
    nf, nb, ns = C.c_int(0), C.c_int(0), C.c_int(0)

    def set_raw(**kw):
        b = _lib.fid_charuco_board()
        b.squares_x, b.squares_y, b.square_length, b.marker_length, b.min_markers, b.check_markers = 5, 7, 0.03, 0.02, 2, 1
        keep = None
        for k, v in kw.items():
            if k == "ids":
                keep = np.ascontiguousarray(v, np.int32)
                b.ids = keep.ctypes.data
            else:
                setattr(b, k, v)
        return lib.fid_set_charuco_boards(det.h, 1, C.byref(b))

    assert set_raw(squares_x=1) == -1 and set_raw(squares_y=1) == -1 and set_raw(squares_x=34, squares_y=34) == -1
    assert set_raw(marker_length=0.03) == -1 and set_raw(square_length=0.0) == -1 and set_raw(min_markers=3) == -1
    assert set_raw(ids=[1] * 17) == -1                      # a repeated id
    assert set_raw(squares_x=30, squares_y=30) == -1        # 450 markers: more than DICT_6X6_250 has
    assert lib.fid_set_charuco_boards(det.h, 17, None) == -1 and lib.fid_set_charuco_boards(det.h, 1, None) == -1
    recs = (_lib.fid_charuco_result * 2)()
    cid = np.zeros(64, np.int32)
    cxy = np.zeros((64, 2), np.float32)
    args = (frame.ctypes.data_as(C.c_void_p), 640, 480, 640 * 3, 0, None, None, None, C.cast(recs, C.c_void_p), cid.ctypes.data_as(C.c_void_p),
            cxy.ctypes.data_as(C.c_void_p))
    assert lib.fid_detect_charuco(det.h, *args) == -1       # no boards set
    assert lib.fid_last_charuco(det.h, 64, C.byref(nf), C.byref(nb), C.byref(ns), None, None, None) == -1
    assert set_raw() == 0
    assert lib.fid_detect_charuco(det.h, *args) == 0 and recs[0].n_corners == 0 and cid[0] == -1
    frames = np.zeros((2, 480, 640, 3), np.uint8)
    det.submit_batch(frames)
    assert set_raw() == -1 and lib.fid_detect_charuco(det.h, *args) == -1  # not while a batch is in flight
    det.collect_batch()
    assert lib.fid_last_charuco(det.h, 0, C.byref(nf), C.byref(nb), C.byref(ns), None, None, None) == 0 and (nf.value, nb.value, ns.value) == (2, 1, 24)
    assert lib.fid_last_charuco(det.h, 23, C.byref(nf), C.byref(nb), C.byref(ns), C.cast(recs, C.c_void_p), cid.ctypes.data_as(C.c_void_p),
                                cxy.ctypes.data_as(C.c_void_p)) == -5
    assert lib.fid_set_charuco_boards(det.h, 0, None) == 0  # off again
    det.close()


GRID = grid_board((2, 2), 0.03, 0.008, [200, 201, 202, 203])


def _frames_with_grid(n, seed):
    """n BGR frames with BOARD_A left, BOARD_B middle and the marker board GRID right; every 3rd frame without any board."""
    rng = np.random.default_rng(seed)
    gb = cv2.aruco.GridBoard((2, 2), 0.03, 0.008, co.DICT, GRID.ids)
    px, margin = 1500.0, 30
    ext = GRID.obj_points.reshape(-1, 3).max(0)
    img = gb.generateImage((int(round(ext[0] * px)) + 2 * margin, int(round(ext[1] * px)) + 2 * margin), marginSize=margin, borderBits=1)
    A = np.array([[1 / px, 0, -margin / px], [0, 1 / px, -margin / px], [0, 0, 1]])
    out = []
    for f in range(n):
        g = np.full((H, W), 128, np.uint8)
        if f % 3 != 2:
            for bi, b in enumerate((BOARD_A, BOARD_B)):
                cvb = co.cv_board(b.size, b.square_length, b.marker_length, b.ids, b.legacy)
                R, t = co.board_pose_in_view(cvb, rng, K_R, W // 3, H, kind="near", centre=(W * (bi + 0.5) / 3, H / 2 + rng.uniform(-40, 40)))
                co.render(g, cvb, R, t, K_R)
            R = co._rot(rng.normal(0, 0.15, 3))
            z = 0.45
            t = z * np.array([(W * 2.5 / 3 - K_R[0, 2]) / K_R[0, 0], (H / 2 - K_R[1, 2]) / K_R[1, 1], 1.0]) - R @ np.array([ext[0] / 2, ext[1] / 2, 0])
            Hm = K_R @ np.column_stack([R[:, 0], R[:, 1], t]) @ A
            warped = cv2.warpPerspective(img, Hm, (W, H), flags=cv2.INTER_LINEAR)
            mask = cv2.warpPerspective(np.full_like(img, 255), Hm, (W, H), flags=cv2.INTER_NEAREST)
            g[mask > 0] = warped[mask > 0]
        out.append(cv2.cvtColor(co.blur_noise(g, rng), cv2.COLOR_GRAY2BGR))
    return np.ascontiguousarray(np.stack(out))


def _check_batch(det, frames, counts, ids, corners, ch):
    """Every (frame, board) of a batch: the single-frame call on the same markers bit for bit, and cv2 on the detector's markers."""
    corners = corners.reshape(len(frames), MAXM, 8)
    n_corners = 0
    for f in range(len(frames)):
        n = int(counts[f])
        single = det.charuco(frames[f], ids[f, :n], corners[f, :n], K_R, D_ZERO)
        gray = cv2.cvtColor(frames[f], cv2.COLOR_BGR2GRAY)
        for bi, ((r1, i1, x1), (r2, i2, x2)) in enumerate(zip(ch[f], single)):
            assert bytes(r1) == bytes(r2) and np.array_equal(i1, i2) and np.array_equal(x1, x2), (f, bi)
            if n:
                check((BOARD_A, BOARD_B)[bi], gray, ids[f, :n], corners[f, :n], K_R, D_ZERO, "batch frame %d board %d" % (f, bi))
            n_corners += int(r1.n_corners)
    return n_corners


def test_two_batches_in_flight_multi_chunk_and_marker_board():
    """Two multi-chunk batches in flight and fid_detect_pose_batch, with two ChArUco boards and a marker board in the same frames."""
    frames = _frames_with_grid(10, 5)
    det = Detector(default_params(dictionary=co.DICT_ID), 0, W, H, 4)  # 3 chunks per 10-frame batch
    det.set_boards([GRID])
    det.set_charuco_boards([BOARD_A, BOARD_B])
    a, b = np.ascontiguousarray(frames[:6]), np.ascontiguousarray(frames[6:])
    det.submit_batch(a, K_R, D_ZERO, FLEN)
    det.submit_batch(b, K_R, D_ZERO, FLEN)  # two batches in flight: each keeps its own records
    got = []
    for part in (a, b):
        counts, ids, corners, _ = det.collect_batch()
        got.append((part, counts, ids, corners, det.last_charuco()))
        assert len(got[-1][-1]) == len(part)
    total = 0
    for part, counts, ids, corners, ch in got:  # fid_detect_charuco only once nothing is in flight
        total += _check_batch(det, part, counts, ids, corners, ch)
    assert total >= 60, total
    counts, ids, corners, _ = det.detect_pose_batch(frames, K_R, D_ZERO, FLEN)
    ch = det.last_charuco()
    _check_batch(det, frames, counts, ids, corners, ch)
    # the marker board is detected in the same frames and its pose solved alongside
    grid = det.last_board_poses()
    assert sum(int(fr[0].status == 1) for fr in grid) >= 5
    det.close()


def test_node_attaches_charuco():
    from fiducials_b200.node import FiducialsNode
    frames = _frames(3, 6, [BOARD_A, BOARD_B])
    plain = FiducialsNode(dictionary=co.DICT_ID, fiducial_len=FLEN, max_width=W, max_height=H, max_batch=2)
    node = FiducialsNode(dictionary=co.DICT_ID, fiducial_len=FLEN, max_width=W, max_height=H, max_batch=2, charuco_boards=[BOARD_A, BOARD_B])
    for nd in (plain, node):
        nd.camInfoCallback(K_R, D_ZERO, "camera")
    fta0 = plain.poseEstimateCallback(plain.imageCallback(frames[0]))
    fta = node.poseEstimateCallback(node.imageCallback(frames[0]))
    assert fta.transforms == fta0.transforms and not hasattr(fta0, "charuco")
    assert [int(r.board) for r, _, _ in fta.charuco] == [0, 1] and all(r.status == 1 and len(i) == r.n_corners > 0 for r, i, _ in fta.charuco)
    batch0, batch = plain.process_batch(frames), node.process_batch(frames)
    for x, y in zip(batch0, batch):
        assert x.transforms == y.transforms and len(y.charuco) == 2
    for (r1, i1, x1), (r2, i2, x2) in zip(batch[0].charuco, fta.charuco):
        assert bytes(r1) == bytes(r2) and np.array_equal(i1, i2) and np.array_equal(x1, x2)
