"""cv2 side of the marker-refinement tests: rendered marker boards and ChArUco boards with damaged markers, cv2's detectMarkers lists,
and cv2.aruco.ArucoDetector.refineDetectedMarkers run board after board as fiducials_b200 runs it."""
import cv2
import numpy as np

from fiducials_b200.board import CharucoBoard
from oracle import aruco_oracle as ao

DICT = cv2.aruco.DICT_6X6_250


def detector(refine=None, **overrides):
    """The project's detector parameters (aruco_oracle) with overrides, and refine = (minRepDistance, errorCorrectionRate,
    checkAllOrders) or None for cv2's defaults."""
    rp = cv2.aruco.RefineParameters(*refine) if refine is not None else cv2.aruco.RefineParameters()
    return cv2.aruco.ArucoDetector(cv2.aruco.getPredefinedDictionary(DICT), ao.reference_detector_params(**overrides), rp)


def cv_board(board):
    """The cv2 board of a fiducials_b200 board: a cv2.aruco.CharucoBoard for a CharucoBoard (refineDetectedMarkers then goes through
    its own class), a generic cv2.aruco.Board otherwise."""
    d = cv2.aruco.getPredefinedDictionary(DICT)
    if isinstance(board, CharucoBoard):
        cb = cv2.aruco.CharucoBoard(board.size, board.square_length, board.marker_length, d, np.asarray(board.ids, np.int32))
        cb.setLegacyPattern(board.legacy)
        return cb
    return cv2.aruco.Board([np.asarray(o, np.float32) for o in board.obj_points], d, np.asarray(board.ids, np.int32))


def detect(det, gray):
    """detectMarkers: ids [n] int32, corners [n,4,2] float32, rejected [m,4,2] float32."""
    corners, ids, rej = det.detectMarkers(cv2.cvtColor(gray, cv2.COLOR_GRAY2BGR))
    ids = np.zeros(0, np.int32) if ids is None else ids.reshape(-1).astype(np.int32)
    corners = np.array(corners, np.float32).reshape(-1, 4, 2)
    rej = np.array(rej, np.float32).reshape(-1, 4, 2)
    return ids, corners, rej


def refine(det, gray, boards, ids, corners, rej, K=None, D=None):
    """refineDetectedMarkers against each board in turn, each call on the lists the previous one returned.  Returns ids, corners,
    the remaining rejected list, per recovered marker its index into the rejected list as first passed and its board, and per board
    whether cv2 raised (that call then changes nothing)."""
    ids, corners, rej = np.asarray(ids, np.int32), np.asarray(corners, np.float32).reshape(-1, 4, 2), np.asarray(rej, np.float32).reshape(-1, 4, 2)
    remaining = list(range(len(rej)))
    rec_idx, rec_board, raised = [], [], []
    bgr = cv2.cvtColor(gray, cv2.COLOR_GRAY2BGR)
    for b, board in enumerate(boards):
        args = [bgr, cv_board(board), tuple(c.reshape(1, 4, 2).copy() for c in corners), ids.reshape(-1, 1).copy(),
                tuple(r.reshape(1, 4, 2).copy() for r in rej)]
        if K is not None:
            args += [np.asarray(K, np.float64), np.asarray(D, np.float64)]
        try:
            c2, i2, r2, rec = det.refineDetectedMarkers(*args)
        except cv2.error:
            raised.append(True)
            continue
        raised.append(False)
        rec = [] if rec is None else np.asarray(rec).reshape(-1).tolist()
        rec_idx += [remaining[k] for k in rec]
        rec_board += [b] * len(rec)
        remaining = [r for k, r in enumerate(remaining) if k not in set(rec)]
        ids = np.zeros(0, np.int32) if i2 is None else np.asarray(i2).reshape(-1).astype(np.int32)
        corners = np.array(c2, np.float32).reshape(-1, 4, 2)
        rej = np.array(r2, np.float32).reshape(-1, 4, 2)
    return ids, corners, rej, rec_idx, rec_board, raised


# ---- rendered boards ------------------------------------------------------------------------------------------------------------
def _rot(v):
    return cv2.Rodrigues(np.asarray(v, np.float64).reshape(3, 1))[0]


def extent(board):
    o = np.asarray(board.obj_points).reshape(-1, 3)
    return o[:, 0].min(), o[:, 1].min(), o[:, 0].max(), o[:, 1].max()


def pose_in_view(board, rng, K, W, H, kind="near"):
    """A pose (R, t) that puts the board's centre in front of the camera: near, far or oblique."""
    x0, y0, x1, y1 = extent(board)
    c = np.array([(x0 + x1) / 2, (y0 + y1) / 2, 0.0])
    ext = max(x1 - x0, y1 - y0)
    f = K[0, 0]
    frac = {"near": (0.5, 0.8), "far": (0.15, 0.3), "oblique": (0.4, 0.7)}[kind]
    tilt = rng.uniform(0.6, 0.9) if kind == "oblique" else rng.uniform(0.0, 0.4)
    z = ext * f / rng.uniform(*frac) / W
    ax = rng.normal(size=3)
    ax[2] = 0.0
    ax /= np.linalg.norm(ax)
    R = _rot(ax * tilt) @ _rot([0.0, 0.0, rng.uniform(-0.4, 0.4)])
    u, v = rng.uniform(0.4 * W, 0.6 * W), rng.uniform(0.4 * H, 0.6 * H)
    t = z * np.array([(u - K[0, 2]) / K[0, 0], (v - K[1, 2]) / K[1, 1], 1.0]) - R @ c
    return R, t


def _homography(R, t, K):
    return np.asarray(K, np.float64) @ np.column_stack([R[:, 0], R[:, 1], t])


def render(gray, board_img, metres_per_px, origin, R, t, K):
    """Warp a printed board image (pixel (u, v) = board point origin + (u, v) * metres_per_px) into gray at pose (R, t), in place."""
    A = np.array([[metres_per_px, 0, origin[0]], [0, metres_per_px, origin[1]], [0, 0, 1]])
    Hm = _homography(R, t, K) @ A
    H, W = gray.shape
    warped = cv2.warpPerspective(board_img, Hm, (W, H), flags=cv2.INTER_LINEAR)
    mask = cv2.warpPerspective(np.full_like(board_img, 255), Hm, (W, H), flags=cv2.INTER_NEAREST)
    gray[mask > 0] = warped[mask > 0]


def render_grid(gray, size, length, sep, R, t, K, ids=None, px=60):
    """cv2.aruco.GridBoard(size, length, sep).generateImage warped into gray."""
    g = cv2.aruco.GridBoard(size, length, sep, cv2.aruco.getPredefinedDictionary(DICT), None if ids is None else np.asarray(ids, np.int32))
    mpp = length / px
    margin = px // 2
    w = int(round((size[0] * length + (size[0] - 1) * sep) / mpp)) + 2 * margin
    h = int(round((size[1] * length + (size[1] - 1) * sep) / mpp)) + 2 * margin
    img = g.generateImage((w, h), marginSize=margin, borderBits=1)
    render(gray, img, mpp, (-margin * mpp, -margin * mpp), R, t, K)


def render_charuco(gray, size, square, marker, R, t, K, ids=None, px=60):
    b = cv2.aruco.CharucoBoard(size, square, marker, cv2.aruco.getPredefinedDictionary(DICT), None if ids is None else np.asarray(ids, np.int32))
    margin = px // 2
    img = b.generateImage((size[0] * px + 2 * margin, size[1] * px + 2 * margin), marginSize=margin, borderBits=1)
    mpp = square / px
    render(gray, img, mpp, (-margin * mpp, -margin * mpp), R, t, K)


def damage(gray, board, k, R, t, K, rng, kind="stripe"):
    """Paint over inner bits of board marker k: "stripe" covers a band of rows of the code, "full" the whole code, "occlude" a
    block across one corner of the marker (its border breaks too)."""
    o = np.asarray(board.obj_points[k], np.float64)
    ms = cv2.aruco.getPredefinedDictionary(DICT).markerSize
    u, v = (o[1] - o[0]) / (ms + 2), (o[3] - o[0]) / (ms + 2)
    if kind == "stripe":
        r0 = int(rng.integers(1, ms - 1))
        quad = [o[0] + u + v * r0, o[0] + u * (ms + 1) + v * r0, o[0] + u * (ms + 1) + v * (r0 + 2), o[0] + u + v * (r0 + 2)]
    elif kind == "full":
        quad = [o[0] + u + v, o[0] + u * (ms + 1) + v, o[0] + (u + v) * (ms + 1), o[0] + u + v * (ms + 1)]
    else:
        quad = [o[2] - 3 * (u + v), o[2] - 3 * v + u, o[2] + u + v, o[2] - 3 * u + v]
    Hm = _homography(R, t, K)
    p = np.array([(Hm @ np.array([q[0], q[1], 1.0])) for q in quad])
    p = p[:, :2] / p[:, 2:]
    cv2.fillConvexPoly(gray, np.round(p * 16).astype(np.int32), int(rng.choice([0, 255, 128])), lineType=cv2.LINE_AA, shift=4)
