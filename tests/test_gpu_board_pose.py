"""One pose per marker board on the device (fid_set_boards, fid_estimate_board_poses, fid_last_board_poses) against
cv2.aruco.Board.matchImagePoints + cv2.solvePnP(SOLVEPNP_ITERATIVE) and the host build of the same arithmetic, and the default outputs
with boards set and without."""
import ctypes as C
import math

import cv2
import numpy as np
import pytest

from fiducials_b200 import _lib, synth
from fiducials_b200.board import grid_board
from fiducials_b200.node import MAXM, Detector, FiducialsNode, default_params
import board_oracle as bo
from test_hostsim_board import hs_board_pose

pytestmark = pytest.mark.gpu

K_SYN, D_REF = synth.camera_for(640, 480)
D_ZERO = np.zeros(5)
DICT_ID = 10  # DICT_6X6_250
FLEN = 0.14


@pytest.fixture(scope="module")
def det640():
    d = Detector(default_params(dictionary=DICT_ID), 0, 640, 480, 2)
    yield d
    d.close()


_stats = {"cases": 0, "identical": 0, "max_host_diff": 0.0}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\ndevice vs host build: %d of %d poses bit-identical, max |difference| %.3g" % (_stats["identical"], _stats["cases"], _stats["max_host_diff"]))


def _check_host_corners(det, cases, K, D):
    for i, (b, ids, corners) in enumerate(cases):
        det.set_boards([b])
        (r,) = det.board_poses(ids, corners, K, D)
        got = bo.record_dict(r)
        assert got["board"] == 0
        bo.assert_matches(got, bo.board_pose(b, ids, corners, K, D), "case %d" % i)
        hs = hs_board_pose(b, ids, corners, K, D)
        assert (got["status"], got["n_markers"], got["n_points"]) == (hs["status"], hs["n_markers"], hs["n_points"])
        diff = max(np.abs(got[k] - hs[k]).max() for k in ("rvec", "tvec", "rotation"))
        diff = max(diff, abs(got["image_error"] - hs["image_error"]))
        same = all(np.array_equal(got[k], hs[k]) for k in ("rvec", "tvec", "rotation")) and got["image_error"] == hs["image_error"]
        _stats["cases"] += 1
        _stats["identical"] += int(same)
        _stats["max_host_diff"] = max(_stats["max_host_diff"], diff)
        # not always bit-identical: the device's sin / cos / acos / exp (Rodrigues, the LM lambda) and the host C library's differ in
        # the last bit for some arguments, and the LM trajectory carries that rounding (measured max 1.4e-12 on an H100)
        assert diff <= 1e-10, ("case %d" % i, got, hs)


@pytest.mark.parametrize("D", [D_REF, D_ZERO], ids=["D_ref", "D_zero"])
@pytest.mark.parametrize("seed", range(2))
def test_host_corners_grid_boards(det640, seed, D):
    _check_host_corners(det640, bo.grid_cases(10 + seed, K_SYN, D, n=15), K_SYN, D)


@pytest.mark.parametrize("D", [D_REF, D_ZERO], ids=["D_ref", "D_zero"])
def test_host_corners_tilted_plane_cube_and_bent(det640, D):
    rng = np.random.default_rng(50)
    cases = []
    for k in range(4):
        b = bo.transformed(grid_board((3, 4), 0.05, 0.012), bo._rot(rng.normal(0, 0.6, 3)), rng.normal(0, 0.3, 3))
        R, t = bo.board_in_view(b, rng, K_SYN, kind=["near", "far", "oblique"][k % 3])
        cases.append((b,) + bo.detections(b, R, t, K_SYN, D, rng, noise=0.3))
    for faces in (2, 3):
        b = bo.cube_board(faces)
        R = bo._rot([rng.uniform(-0.5, -0.3), rng.uniform(-0.8, -0.4), 0.1])
        cases.append((b,) + bo.detections(b, R, np.array([0.05, -0.02, 1.2]), K_SYN, D, rng, noise=0.2))
    b = bo.bent_marker()
    cases.append((b,) + bo.detections(b, bo._rot([math.pi, 0.1, 0.0]), np.array([0.02, -0.01, 0.6]), K_SYN, D, rng, noise=0.1))
    _check_host_corners(det640, cases, K_SYN, D)
    assert bo.board_pose(*cases[-1], K_SYN, D)["status"] == -1


def test_host_corners_empty_and_off_board(det640):
    b = grid_board((3, 3), 0.05, 0.01)
    det640.set_boards([b, grid_board((2, 2), 0.05, 0.01, [40, 41, 42, 43])])
    for ids in ([], [100, 200], [41, 200, 41]):
        corners = np.random.default_rng(len(ids)).uniform(100, 300, (len(ids), 4, 2)).astype(np.float32)
        recs = [bo.record_dict(r) for r in det640.board_poses(ids, corners, K_SYN, D_ZERO)]
        assert [r["board"] for r in recs] == [0, 1]
        assert recs[0]["status"] == 0 and recs[0]["n_points"] == 0 and not np.any(recs[0]["rvec"]) and recs[0]["image_error"] == 0.0
        assert recs[1]["n_markers"] == 2 * (ids.count(41) > 0)


# ---- rendered frames ----------------------------------------------------------------------------------------------------------
W, H = 1280, 720
K_R, _ = synth.camera_for(W, H)
BOARD_A = grid_board((4, 3), 0.04, 0.01)                               # ids 0..11
BOARD_B = grid_board((3, 3), 0.035, 0.008, list(range(100, 109)))      # ids 100..108
_PX_PER_M, _MARGIN = 2500.0, 40


_GRID = {id(BOARD_A): ((4, 3), 0.04, 0.01), id(BOARD_B): ((3, 3), 0.035, 0.008)}


def _render(frame, board, R, t):
    """cv2.aruco.GridBoard.generateImage of the board, warped into the gray frame at pose (R, t) (no distortion)."""
    size, length, sep = _GRID[id(board)]
    gb = cv2.aruco.GridBoard(size, length, sep, bo.DICT, board.ids)
    ext = board.obj_points.reshape(-1, 3).max(0)
    bw, bh = int(round(ext[0] * _PX_PER_M)) + 2 * _MARGIN, int(round(ext[1] * _PX_PER_M)) + 2 * _MARGIN
    img = gb.generateImage((bw, bh), marginSize=_MARGIN, borderBits=1)
    A = np.array([[1 / _PX_PER_M, 0, -_MARGIN / _PX_PER_M], [0, 1 / _PX_PER_M, -_MARGIN / _PX_PER_M], [0, 0, 1]])  # image px -> board metres
    Hm = K_R @ np.column_stack([R[:, 0], R[:, 1], t]) @ A
    warped = cv2.warpPerspective(img, Hm, (W, H), flags=cv2.INTER_LINEAR)
    mask = cv2.warpPerspective(np.full_like(img, 255), Hm, (W, H), flags=cv2.INTER_NEAREST)
    frame[mask > 0] = warped[mask > 0]


def _pose(rng, u, v, z):
    """A board facing the camera (its x right, y down as printed), tilted by up to ~20 degrees."""
    R = bo._rot(rng.normal(0, 0.2, 3) * np.array([1, 1, 0.5]))
    t = z * np.array([(u - K_R[0, 2]) / K_R[0, 0], (v - K_R[1, 2]) / K_R[1, 1], 1.0]) - R @ np.array([0.08, 0.06, 0.0])
    return R, t


def rendered_frames(n, seed=0):
    """n BGR frames: both boards (A left, B right), some markers painted over, every 4th frame without any board marker.
    Returns frames [n,H,W,3] and the rendering poses {(frame, board): (R, t)}."""
    rng = np.random.default_rng(seed)
    frames, poses = [], {}
    for f in range(n):
        fr = np.full((H, W), 128, np.uint8)
        if f % 4 != 3:
            for bi, (board, u) in enumerate(((BOARD_A, 0.3 * W), (BOARD_B, 0.72 * W))):
                R, t = _pose(rng, u + rng.uniform(-40, 40), 0.5 * H + rng.uniform(-60, 60), rng.uniform(0.45, 0.8))
                _render(fr, board, R, t)
                poses[(f, bi)] = (R, t)
                if f % 4 == 1:  # paint over two markers
                    for k in rng.choice(len(board), 2, replace=False):
                        q = bo.project(board.obj_points[k], R, t, K_R, D_ZERO).reshape(4, 2)
                        cv2.fillConvexPoly(fr, np.round((q - q.mean(0)) * 1.15 + q.mean(0)).astype(np.int32), 255)
        frames.append(cv2.cvtColor(fr, cv2.COLOR_GRAY2BGR))
    return np.ascontiguousarray(np.stack(frames)), poses


def _check_batch(counts, ids, corners, recs, poses, first=0):
    n_solved = 0
    for f in range(len(counts)):
        n = int(counts[f])
        for bi, board in enumerate((BOARD_A, BOARD_B)):
            got = bo.record_dict(recs[f][bi])
            assert got["board"] == bi
            ref = bo.board_pose(board, ids[f, :n], corners[f, :n], K_R, D_ZERO)  # the oracle on the device's own detections
            bo.assert_matches(got, ref, "frame %d board %d" % (first + f, bi))
            if (first + f, bi) in poses and got["status"] == 1:
                R, t = poses[(first + f, bi)]
                Rg = cv2.Rodrigues(got["rvec"].reshape(3, 1))[0]
                assert np.degrees(np.arccos(np.clip((np.trace(Rg.T @ R) - 1) / 2, -1, 1))) < 2.0  # loose: the rendering pose
                assert np.linalg.norm(got["tvec"] - t) < 0.03 * np.linalg.norm(t)
                n_solved += 1
            if (first + f) % 4 == 3:
                assert got["status"] == 0 and got["n_markers"] == 0
    return n_solved


def test_rendered_batches_submit_collect_and_detect_pose_batch():
    frames, poses = rendered_frames(12, seed=1)
    det = Detector(default_params(dictionary=DICT_ID), 0, W, H, 4)  # 3 chunks per 12-frame batch
    det.set_boards([BOARD_A, BOARD_B])
    a, b = np.ascontiguousarray(frames[:8]), np.ascontiguousarray(frames[8:])
    det.submit_batch(a, K_R, D_ZERO, FLEN)
    det.submit_batch(b, K_R, D_ZERO, FLEN)  # two batches in flight: each keeps its own records
    n_solved, first = 0, 0
    for part in (a, b):
        counts, ids, corners, _ = det.collect_batch()
        recs = det.last_board_poses()
        assert len(recs) == len(part) and all(len(r) == 2 for r in recs)
        n_solved += _check_batch(counts, ids, corners.reshape(len(part), MAXM, 8), recs, poses, first)
        first += len(part)
    assert n_solved >= 14, n_solved
    # the synchronous batch call: the same records, and those of the host-corner call on the same detections bit for bit
    counts, ids, corners, _ = det.detect_pose_batch(frames, K_R, D_ZERO, FLEN)
    recs = det.last_board_poses()
    _check_batch(counts, ids, corners.reshape(len(frames), MAXM, 8), recs, poses)
    for f in range(len(frames)):
        lst = det.board_poses(ids[f, : counts[f]], corners[f, : counts[f]], K_R, D_ZERO)
        assert [bytes(r) for r in lst] == [bytes(r) for r in recs[f]]
    det.close()


def test_default_outputs_unchanged_by_boards():
    frames, _ = rendered_frames(6, seed=2)
    det = Detector(default_params(dictionary=DICT_ID), 0, W, H, 4)
    det.set_pose_hypotheses(True)
    res = []
    for boards in ([], [BOARD_A, BOARD_B], []):
        det.set_boards(boards)
        det.submit_batch(frames, K_R, D_ZERO, FLEN)
        counts, ids, corners, tfs = det.collect_batch()
        res.append((counts.tobytes(), ids.tobytes(), corners.tobytes(), bytes(tfs), bytes(det.last_pose_hypotheses())))
    assert res[0] == res[1] == res[2]
    assert np.frombuffer(res[0][0], np.int32).sum() >= 40
    det.close()


def test_node_attaches_board_poses():
    frames, poses = rendered_frames(3, seed=3)
    plain = FiducialsNode(dictionary=DICT_ID, fiducial_len=FLEN, max_width=W, max_height=H, max_batch=2)
    node = FiducialsNode(dictionary=DICT_ID, fiducial_len=FLEN, max_width=W, max_height=H, max_batch=2, boards=[BOARD_A, BOARD_B])
    for n in (plain, node):
        n.camInfoCallback(K_R, D_ZERO, "camera")
    fta0 = plain.poseEstimateCallback(plain.imageCallback(frames[0]))
    fta = node.poseEstimateCallback(node.imageCallback(frames[0]))
    assert fta.transforms == fta0.transforms and not hasattr(fta0, "board_poses")
    assert [r.board for r in fta.board_poses] == [0, 1] and all(r.status == 1 for r in fta.board_poses)
    batch0, batch = plain.process_batch(frames), node.process_batch(frames)
    for a, b in zip(batch0, batch):
        assert a.transforms == b.transforms and len(b.board_poses) == 2
    assert [bytes(r) for r in batch[0].board_poses] == [bytes(r) for r in fta.board_poses]


def test_errors():
    frames, _ = rendered_frames(2, seed=4)
    det = Detector(default_params(dictionary=DICT_ID), 0, W, H, 2)
    lib, nf, nb = det.lib, C.c_int(0), C.c_int(0)
    buf = (_lib.fid_board_pose * 8)()
    cam = _lib.fid_camera()
    for i, v in enumerate(K_R.reshape(9)):
        cam.K[i] = float(v)
    one_id = np.zeros(1, np.int32)
    one_c = np.zeros(8, np.float32)

    def set_raw(boards):
        keep = [(np.ascontiguousarray(i, np.int32), np.ascontiguousarray(o, np.float32)) for i, o in boards]
        arr = (_lib.fid_board * max(len(keep), 1))()
        for k, (i, o) in enumerate(keep):
            arr[k].n_markers, arr[k].ids, arr[k].obj_points = len(i), i.ctypes.data, o.ctypes.data
        return lib.fid_set_boards(det.h, len(keep), C.cast(arr, C.c_void_p))

    ok = (BOARD_A.ids, BOARD_A.obj_points)
    assert set_raw([ok] * 17) == -1                                               # more than FID_MAX_BOARDS
    assert set_raw([(np.arange(4097), np.zeros((4097, 4, 3)))]) == -1             # more than 4096 markers
    assert set_raw([(np.zeros(0), np.zeros((0, 4, 3)))]) == -1                    # no marker
    assert set_raw([(BOARD_A.ids, np.where(np.arange(12)[:, None, None] == 3, np.inf, BOARD_A.obj_points))]) == -1  # non-finite
    assert set_raw([(np.array([1, 2, 1]), np.zeros((3, 4, 3)))]) == -1            # a repeated id within one board
    assert lib.fid_set_boards(det.h, -1, None) == -1 and lib.fid_set_boards(det.h, 1, None) == -1
    # no boards set: the host-corner call has nothing to estimate
    assert lib.fid_estimate_board_poses(det.h, 1, one_id.ctypes.data_as(C.c_void_p), one_c.ctypes.data_as(C.c_void_p), C.byref(cam), C.cast(buf, C.c_void_p)) == -1
    # a batch without boards -> fid_last_board_poses refuses
    det.submit_batch(frames, K_R, D_ZERO, FLEN)
    det.collect_batch()
    assert lib.fid_last_board_poses(det.h, 8, C.byref(nf), C.byref(nb), C.cast(buf, C.c_void_p)) == -1
    # not while a batch is in flight
    det.submit_batch(frames, K_R, D_ZERO, FLEN)
    assert set_raw([ok]) == -1
    det.collect_batch()
    assert set_raw([ok, (BOARD_B.ids, BOARD_B.obj_points)]) == 0
    # boards set, but a batch without a camera: no pose, no records
    det.submit_batch(frames)
    det.collect_batch()
    assert lib.fid_last_board_poses(det.h, 8, C.byref(nf), C.byref(nb), C.cast(buf, C.c_void_p)) == -1
    # with a camera: FID_ERR_CAPACITY (nothing written) when max_boards < the board count, then the records
    det.submit_batch(frames, K_R, D_ZERO, FLEN)
    det.collect_batch()
    for r in buf:
        r.board = -7
    assert lib.fid_last_board_poses(det.h, 1, C.byref(nf), C.byref(nb), C.cast(buf, C.c_void_p)) == -5
    assert all(r.board == -7 for r in buf)
    assert lib.fid_last_board_poses(det.h, 2, C.byref(nf), C.byref(nb), None) == 0 and (nf.value, nb.value) == (2, 2)
    assert lib.fid_last_board_poses(det.h, 2, C.byref(nf), C.byref(nb), C.cast(buf, C.c_void_p)) == 0
    assert [buf[k].board for k in range(4)] == [0, 1, 0, 1]
    # the host-corner call: sizes out of range
    for n in (-1, 257):
        assert lib.fid_estimate_board_poses(det.h, n, one_id.ctypes.data_as(C.c_void_p), one_c.ctypes.data_as(C.c_void_p), C.byref(cam), C.cast(buf, C.c_void_p)) == -1
    assert lib.fid_estimate_board_poses(det.h, 1, one_id.ctypes.data_as(C.c_void_p), one_c.ctypes.data_as(C.c_void_p), None, C.cast(buf, C.c_void_p)) == -1
    assert set_raw([]) == 0  # off again
    det.close()
