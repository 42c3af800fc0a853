"""Seeded dense calibration-target frames: a marker GridBoard or a ChArUco board that fills the frame, rendered by cv2 and seen
through a mild perspective warp and a blur.  Each case is picked for the number of raw quad candidates it gives under the oracle
(oracle.aruco_oracle.quad_candidates), so that together they cross the sizes at which the grouping and output kernels switch paths:

    raw candidates   <= 614 close-pair matrix in shared memory, > 614 in global memory        (k_sort_group)
                     <= 1536 sorted quads in shared memory, > 1536 read from global memory      (k_sort_group)
                     > 2048 three and four matrix words per lane in pass 1                      (k_sort_group)
                     > 4096 clamped at the per-frame capacity: FID_ERR_CAPACITY                 (k_approx, k_sort_group)
    selected         > 512 past the per-frame capacity: FID_ERR_CAPACITY                        (k_sort_group, k_finish)
    markers          > 256 past the per-frame capacity: FID_ERR_CAPACITY, the first 256 written (k_finish)

tests/test_hostsim_dense.py pins every case's band on the CPU; tests/test_gpu_dense_frames.py runs them on the device."""
import cv2
import numpy as np

# the windows that give many markers per raw candidate: 4 scales instead of 13
FEW_SCALES = dict(adaptiveThreshWinSizeMin=3, adaptiveThreshWinSizeMax=15, adaptiveThreshWinSizeStep=4)

# name -> (kind, frame W, H, board cols, rows, dictionary, detector parameter overrides, seed, inverted)
CASES = {}

# bands of the raw-candidate count (inclusive) and the band each case lands in
BANDS = {"le614": (0, 614), "615_1536": (615, 1536), "1537_2048": (1537, 2048), "2049_3072": (2049, 3072), "3073_4096": (3073, 4096),
         "gt4096": (4097, 1 << 30)}


def case(name, kind, W, H, cols, rows, dict_id, band, seed=0, params=None, inverted=False):
    CASES[name] = dict(kind=kind, W=W, H=H, cols=cols, rows=rows, dict_id=dict_id, band=band, seed=seed, params=dict(params or {}), inverted=inverted)


def oracle_params(name):
    """The oracle's parameter dict for the case (REFERENCE_PARAMS with the case's overrides)."""
    from oracle import aruco_oracle as ao

    return dict(ao.REFERENCE_PARAMS, **CASES[name]["params"])


# one case per raw-candidate band, default windows (3..53 step 4, 13 scales), DICT_5X5_1000
case("grid_6x4", "grid", 640, 480, 6, 4, 7, "le614")  # 24 markers
case("grid_10x6", "grid", 1280, 720, 10, 6, 7, "615_1536")  # 60 markers
case("grid_14x8", "grid", 1920, 1080, 14, 8, 7, "1537_2048")  # 112 markers
case("grid_16x9", "grid", 1920, 1080, 16, 9, 7, "2049_3072")  # 144 markers
case("grid_20x12", "grid", 1920, 1080, 20, 12, 7, "3073_4096")  # 240 markers
# detectInvertedMarker: the same board white on black
case("grid_14x8_inverted", "grid", 1920, 1080, 14, 8, 7, "2049_3072", inverted=True)
# the per-frame marker and selected-candidate capacities
case("grid_16x16", "grid", 1920, 1080, 16, 16, 7, "3073_4096")  # exactly 256 markers
case("grid_22x13", "grid", 1920, 1080, 22, 13, 7, "3073_4096")  # 286 markers
case("grid_28x16_few", "grid", 1920, 1080, 28, 16, 3, "1537_2048", params=FEW_SCALES)  # 448 markers, DICT_4X4_1000
case("grid_32x18_few", "grid", 1920, 1080, 32, 18, 3, "2049_3072", params=dict(FEW_SCALES, minMarkerPerimeterRate=0.05))  # 576 markers
# past the raw-candidate capacity: with more markers than fit, and with fewer (a 4K frame of 252 markers)
case("grid_24x14", "grid", 1920, 1080, 24, 14, 7, "gt4096")  # 336 markers
case("grid_18x14_4k", "grid", 3840, 2160, 18, 14, 7, "gt4096")  # 252 markers
# board stages past one 128-wide stride: a ChArUco board of 18 x 12 squares (108 markers, 187 chessboard corners), DICT_6X6_250
case("charuco_18x12", "charuco", 1920, 1080, 18, 12, 10, "3073_4096")

# cv2's marker count of every case (each finds every marker rendered)
MARKERS = {"grid_6x4": 24, "grid_10x6": 60, "grid_14x8": 112, "grid_16x9": 144, "grid_20x12": 240, "grid_14x8_inverted": 112, "grid_16x16": 256,
           "grid_22x13": 286, "grid_28x16_few": 448, "grid_32x18_few": 576, "grid_24x14": 336, "grid_18x14_4k": 252, "charuco_18x12": 108}


def _warp(img, rng, bg):
    """A mild perspective: every image corner moves by up to 2 % of the frame, then a blur of sigma 0.8."""
    H, W = img.shape
    src = np.float32([[0, 0], [W, 0], [W, H], [0, H]])
    dst = src + rng.uniform(-0.02, 0.02, (4, 2)).astype(np.float32) * np.float32([W, H])
    M = cv2.getPerspectiveTransform(src, dst)
    out = cv2.warpPerspective(img, M, (W, H), flags=cv2.INTER_LINEAR, borderValue=int(bg))
    return cv2.GaussianBlur(out, (0, 0), 0.8)


def board(c):
    """The cv2 board of a case (a case name or its CASES entry)."""
    c = CASES[c] if isinstance(c, str) else c
    d = cv2.aruco.getPredefinedDictionary(c["dict_id"])
    if c["kind"] == "grid":
        return cv2.aruco.GridBoard((c["cols"], c["rows"]), 0.04, 0.01, d)
    return cv2.aruco.CharucoBoard((c["cols"], c["rows"]), 0.04, 0.03, d)


def render(name):
    """(bgr H x W x 3 uint8, the rendered ids as a set).  The board fills the frame up to a small margin."""
    c = CASES[name]
    W, H = c["W"], c["H"]
    b = board(c)
    m = max(W, H) // 40
    bw, bh = float(c["cols"]), float(c["rows"])
    if c["kind"] == "grid":  # the grid's extent: cols markers and cols - 1 separations
        bw, bh = bw * 0.05 - 0.01, bh * 0.05 - 0.01
    s = min((W - 2 * m) / bw, (H - 2 * m) / bh)
    w, h = int(bw * s), int(bh * s)
    img = np.full((H, W), 255, np.uint8)
    y0, x0 = (H - h) // 2, (W - w) // 2
    img[y0 : y0 + h, x0 : x0 + w] = b.generateImage((w, h), marginSize=0, borderBits=1)
    if c["inverted"]:
        img = 255 - img
    rng = np.random.default_rng(c["seed"])
    g = _warp(img, rng, 0 if c["inverted"] else 255)
    return np.ascontiguousarray(np.repeat(g[:, :, None], 3, axis=2)), set(np.asarray(b.getIds()).reshape(-1).tolist())


def camera(name):
    c = CASES[name]
    W, H = c["W"], c["H"]
    K = np.array([[1.1 * W, 0, W / 2.0], [0, 1.1 * W, H / 2.0], [0, 0, 1]])
    return K, np.array([0.02, -0.01, 0.0, 0.0, 0.0])
