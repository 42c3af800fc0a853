"""Frames on which detectMarkers' rejectedImgPoints is compared with cv2 4.13 (tests/test_hostsim_rejected.py on the CPU,
tests/test_gpu_batch_refine.py on the device): the synthetic configurations, markers sliding out of the frame, a marker nested inside
a marker, and rendered boards with damaged markers."""
import cv2
import numpy as np

from fiducials_b200 import synth
from fiducials_b200.board import grid_board
from oracle import aruco_oracle as ao
import marker_refine_oracle as mo

W, H = 640, 480
K_SYN, D_REF = synth.camera_for(W, H)


def cv2_lists(bgr, dict_id, **overrides):
    """cv2's detectMarkers with the project's parameters: ids [n] int32, corners [n,4,2], rejected [m,4,2] float32."""
    det = cv2.aruco.ArucoDetector(cv2.aruco.getPredefinedDictionary(dict_id), ao.reference_detector_params(**overrides))
    corners, ids, rej = det.detectMarkers(bgr)
    ids = np.zeros(0, np.int32) if ids is None else ids.reshape(-1).astype(np.int32)
    return ids, np.array(corners, np.float32).reshape(-1, 4, 2), np.array(rej, np.float32).reshape(-1, 4, 2)


def synthetic_frames():
    """(name, bgr, dictionary) of the C1/C2/C3 configurations."""
    for cfg, seed in [("C1", 0), ("C1", 1), ("C1", 2), ("C2", 0), ("C2", 1), ("C3", 0), ("C3", 5)]:
        bgr, _, _, _, d = synth.make_config_frame(cfg, seed)
        yield "%s/%d" % (cfg, seed), bgr, d


def border_frames():
    """C1 frame 0 shifted until its rightmost marker leaves the frame (the frames of test_border_rule_matches_cv2)."""
    bgr, truth, _, _, d = synth.make_config_frame("C1", 0)
    right = np.array([q for _, q in truth])[:, :, 0].max()
    for shift in range(int(640 - right) - 6, int(640 - right) + 8):
        fr = np.roll(bgr, shift, axis=1)
        fr[:, :shift] = 190
        yield "border/%d" % shift, np.ascontiguousarray(fr), d


def nested_frames():
    """A marker inside a white cell of a bigger marker, alone and with a second depth-1 candidate (test_gpu_parity)."""
    from test_gpu_parity import _nested_marker_frames

    for i, fr in enumerate(_nested_marker_frames()):
        yield "nested/%d" % i, np.ascontiguousarray(fr), 10


def damaged_board(seed, kind="near", size=(5, 4), n_damaged=3):
    """A rendered GridBoard with damaged markers (marker_refine_oracle), gray [H, W], and the board."""
    rng = np.random.default_rng(seed)
    board = grid_board(size, 0.04, 0.01)
    R, t = mo.pose_in_view(board, rng, K_SYN, W, H, kind)
    g = np.full((H, W), 128, np.uint8)
    mo.render_grid(g, size, 0.04, 0.01, R, t, K_SYN)
    for k in rng.choice(len(board.ids), min(n_damaged, len(board.ids)), replace=False):
        mo.damage(g, board, int(k), R, t, K_SYN, rng, ("stripe", "stripe", "full", "occlude")[int(rng.integers(4))])
    return board, cv2.GaussianBlur(g, (3, 3), 0.8)


def damaged_frames(n=12):
    for seed in range(n):
        kind = ("near", "far", "oblique")[seed % 3]
        _, g = damaged_board(seed, kind, ((5, 4), (7, 5), (3, 3))[seed % 3])
        yield "damaged/%d" % seed, cv2.cvtColor(g, cv2.COLOR_GRAY2BGR), mo.DICT


def _pose_at(board, rng, u, frac):
    """A pose that puts the board's centre at image column u, its larger side `frac` of the image width, slightly tilted."""
    x0, y0, x1, y1 = mo.extent(board)
    c = np.array([(x0 + x1) / 2, (y0 + y1) / 2, 0.0])
    z = max(x1 - x0, y1 - y0) * K_SYN[0, 0] / frac / W
    ax = rng.normal(size=3)
    ax[2] = 0.0
    ax /= np.linalg.norm(ax)
    R = mo._rot(ax * rng.uniform(0.0, 0.35)) @ mo._rot([0.0, 0.0, rng.uniform(-0.3, 0.3)])
    v = rng.uniform(0.45 * H, 0.55 * H)
    return R, z * np.array([(u - K_SYN[0, 2]) / K_SYN[0, 0], (v - K_SYN[1, 2]) / K_SYN[1, 1], 1.0]) - R @ c


def grid_and_charuco(seed):
    """A 3x3 GridBoard (ids 50..58, one marker damaged) on the left and a 5x4 ChArUco board (ids 0..9, two markers damaged) on the
    right of one gray frame: (grid, charuco, gray)."""
    from fiducials_b200.board import charuco_board

    rng = np.random.default_rng(seed)
    ids = list(range(50, 59))
    grid = grid_board((3, 3), 0.04, 0.01, ids)
    ch = charuco_board((5, 4), 0.04, 0.03)
    g = np.full((H, W), 128, np.uint8)
    Rg, tg = _pose_at(grid, rng, 0.24 * W, 0.38)
    mo.render_grid(g, (3, 3), 0.04, 0.01, Rg, tg, K_SYN, ids)
    Rc, tc = _pose_at(ch, rng, 0.72 * W, 0.5)
    mo.render_charuco(g, (5, 4), 0.04, 0.03, Rc, tc, K_SYN)
    for k in rng.choice(9, 1, replace=False):
        mo.damage(g, grid, int(k), Rg, tg, K_SYN, rng, "stripe")
    for k in rng.choice(10, 2, replace=False):
        mo.damage(g, ch, int(k), Rc, tc, K_SYN, rng, "stripe")
    return grid, ch, cv2.GaussianBlur(g, (3, 3), 0.8)
