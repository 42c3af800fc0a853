"""Seeded frames for the contour stage: the start-crack queue the threshold kernels fill, the border walk's rounds (k_walk), the
contour emission (k_emit) and the polygon fit (k_approx*).  No stored images: every frame is generated here.

Start cracks.  halo_row_starts (contour_walk.cuh) reports a left crack only where `mid & ~mid_l`, so a plane holds at most one left
and one right crack per two pixels of a row: with n_scales planes at most n_scales / 2 per pixel and side (6.5 with the default 13
windows).  fid_create sizes the queue for 3 per pixel and side (6 W H + 65536, half per side).  Uniform noise and natural scenes stay
far below (about 1.6 per side); a 1-pixel checkerboard or dither puts the same pattern into all 13 planes and reaches the bound.  Such
a frame overflows the queue; the device then rescans the stored planes in groups of scales that provably fit and replays the walk
(kernels_contour.cuh, k_rescan_starts), so the frame's result does not change.

Length filter.  The detector and the oracle run with the reference's minMarkerPerimeterRate 0.1 and maxMarkerPerimeterRate 4.0
(oracle.aruco_oracle.REFERENCE_PARAMS): contours of min_len = (int)(0.1 max(W, H)) to max_len = (int)(4 max(W, H)) points are walked to
the end and fitted.

Chains and points.  max_chains = 65536 in-range contours per frame slot and max_points = 4 W H + 65536 contour points, both sized from
the handle's maximum frame.  65536 in-range contours need at least 65536 min_len points, which exceeds 4 W H + 65536 whenever the
frame fills the handle and its shorter side is under 1639 pixels (6553.6 max(W, H) > 4 W H): on such a frame the point capacity is
always reached first.  The chain capacity alone is reached by a frame smaller than its handle -- "segments": 1280 x 720 in a
3840 x 2160 handle, 1-pixel line segments of 66 pixels (130-point contours, min_len 128, not 4-gons), 82 000 in-range contours and
11 M points.  The point capacity is reached by long in-range contours on every plane: 1-pixel lines two pixels apart give every
plane H / 2 contours of 2 (W - 1) points -- "lines".  Both are legitimate frames whose status is FID_ERR_CAPACITY;
tests/test_gpu_contour_stage.py checks that every marker returned is cv2's.

Every case declares the bands its counters land in; tests/test_hostsim_contour_capacity.py pins them on the CPU."""
import functools

import cv2
import numpy as np

DICT = 7  # DICT_5X5_1000
HALO_T = 30  # FID_HALO_T: interior pixels of a halo tile per row / column
SIZES = {"vga": (640, 480), "fhd": (1920, 1080), "uhd": (3840, 2160)}
TEXTURES = ("checker1", "dither1", "checker2", "noise")

# name -> dict(W, H, kind, texture / layout / extra, seed); filled by case()
CASES = {}


def case(name, W, H, kind, **kw):
    CASES[name] = dict(W=W, H=H, kind=kind, **kw)


# ---- fine textures: full frame (markers on white pads) and left half (markers on the flat right half) ---------------------------
for _t in TEXTURES:
    for _s, (_w, _h) in SIZES.items():
        for _layout in ("full", "half"):
            case(f"{_t}_{_layout}_{_s}", _w, _h, "texture", texture=_t, layout=_layout, seed=11)
# ---- the walk rounds (plan 8, 64, 512, persistent) ----------------------------------------------------------------------------------
case("spiral_fhd", 1920, 1080, "spiral", seed=3)  # one contour of ~7 000 points: only the persistent round decides it
case("serpentine_fhd", 1920, 1080, "serpentine", seed=4)  # a contour past max_len next to four in-range markers
# ---- halo tiling: tile seams, frame borders, frame sizes one pixel either side of a tile multiple -------------------------------
for _w, _h in ((599, 449), (600, 450), (601, 451), (1919, 1079), (1921, 1081)):
    case(f"seams_{_w}x{_h}", _w, _h, "seams", seed=5)
case("borders_fhd", 1920, 1080, "borders", seed=6)
# ---- the length filter: contours of exactly min_len - 1, min_len, max_len and max_len + 1 points -----------------------------------
case("length_min_vga", 640, 480, "length_min", seed=7)
case("length_max_vga", 640, 480, "length_max", seed=8)
# ---- chain and point capacities ------------------------------------------------------------------------------------------------------
case("segments_hd_in_uhd", 1280, 720, "segments", seed=9, handle=(3840, 2160))
case("lines_fhd", 1920, 1080, "lines", seed=10)


def handle(name):
    """(max width, max height) of the handle a case runs in: its own size unless it says otherwise."""
    c = CASES[name]
    return c.get("handle", (c["W"], c["H"]))


def min_len(W, H):
    from oracle.aruco_oracle import REFERENCE_PARAMS

    return int(REFERENCE_PARAMS["minMarkerPerimeterRate"] * max(W, H))


def max_len(W, H):
    from oracle.aruco_oracle import REFERENCE_PARAMS

    return int(REFERENCE_PARAMS["maxMarkerPerimeterRate"] * max(W, H))


def texture(kind, H, W, seed):
    y, x = np.mgrid[0:H, 0:W]
    if kind == "checker1":
        return (((x + y) & 1) * 255).astype(np.uint8)
    if kind == "dither1":  # low contrast: 90 / 160
        return np.where((x + y) & 1, 160, 90).astype(np.uint8)
    if kind == "checker2":
        return ((((x >> 1) + (y >> 1)) & 1) * 255).astype(np.uint8)
    return np.random.default_rng(seed).integers(0, 256, (H, W), dtype=np.uint8)


def marker(mid, side):
    return cv2.aruco.generateImageMarker(cv2.aruco.getPredefinedDictionary(DICT), mid, side)


def _paste(img, mid, x0, y0, side, pad=0):
    """A marker with `pad` pixels of white around it (its quiet zone on a textured background)."""
    if pad:
        img[y0 - pad : y0 + side + pad, x0 - pad : x0 + side + pad] = 255
    img[y0 : y0 + side, x0 : x0 + side] = marker(mid, side)


def _four_markers(img, x_lo, x_hi, H, rng, pad):
    """Four markers in a 2 x 2 grid inside columns [x_lo, x_hi): returns their ids."""
    side = int(min(x_hi - x_lo, H) / 4.5)
    ids = [int(v) for v in rng.choice(1000, 4, replace=False)]
    cw, ch = (x_hi - x_lo) // 2, H // 2
    for k, mid in enumerate(ids):
        cx, cy = x_lo + cw * (k % 2) + cw // 2, ch * (k // 2) + ch // 2
        _paste(img, mid, cx - side // 2, cy - side // 2, side, pad)
    return set(ids)


def _spiral(img, cx, cy, r_max, gap, thick):
    """A square spiral of black lines drawn from the centre outwards: one connected curve."""
    pts = [(cx, cy)]
    r, d = gap, 0
    while r < r_max:
        x, y = pts[-1]
        dx, dy = [(1, 0), (0, 1), (-1, 0), (0, -1)][d % 4]
        pts.append((x + dx * r, y + dy * r))
        if d % 2:
            r += gap
        d += 1
    cv2.polylines(img, [np.array(pts, np.int32)], False, 0, thick)


def _render(c):
    W, H = c["W"], c["H"]
    rng = np.random.default_rng(c["seed"])
    kind = c["kind"]
    img = np.full((H, W), 205, np.uint8)
    ids = set()
    if kind == "texture":
        if c["layout"] == "full":
            img[:] = texture(c["texture"], H, W, c["seed"])
            ids = _four_markers(img, 0, W, H, rng, pad=max(8, H // 40))
        else:
            img[:, : W // 2] = texture(c["texture"], H, W // 2, c["seed"])
            ids = _four_markers(img, W // 2, W, H, rng, pad=0)
    elif kind == "spiral":
        _spiral(img, W // 2, H // 2, 300, 24, 3)
        ids = set()
        for k, (x0, y0) in enumerate(((80, 80), (W - 330, 80), (80, H - 330), (W - 330, H - 330))):
            mid = int(rng.integers(0, 1000))
            _paste(img, mid, x0, y0, 240)
            ids.add(mid)
    elif kind == "serpentine":
        # a 2-pixel serpentine of 16 runs across the middle third: one contour of ~2 * 16 * 1300 points > max_len = 7680
        pts = []
        for k in range(16):
            y = 380 + 20 * k
            pts += [(300, y), (1600, y)] if k % 2 == 0 else [(1600, y), (300, y)]
        cv2.polylines(img, [np.array(pts, np.int32)], False, 0, 2)
        ids = _four_markers(img, 0, W, 340, rng, pad=0)
    elif kind == "seams":
        # markers whose outer edges fall on x, y = 0, 1, 29 (mod 30) and blobs cut by every tile seam
        for k, off in enumerate((0, 1, 29)):
            side = 150
            x0, y0 = 30 * (1 + 6 * k) + off, 30 * 2 + off
            mid = int(rng.integers(0, 1000))
            _paste(img, mid, x0, y0, side)
            ids.add(mid)
        for k in range(60):
            x0 = 30 * int(rng.integers(0, W // 30)) + int(rng.choice([-2, -1, 0, 1, 2]))
            y0 = 30 * int(rng.integers(8, H // 30)) + int(rng.choice([-2, -1, 0, 1, 2]))
            w, h = int(rng.integers(3, 70)), int(rng.integers(3, 70))
            cv2.rectangle(img, (x0, y0), (x0 + w, y0 + h), int(rng.choice([0, 40])), int(rng.choice([-1, 1, 2])))
        img[:, -1] = 0  # the last column and row: contours along the frame's right and bottom borders whatever W mod 30
        img[-1, :] = 0
    elif kind == "borders":
        # markers flush with each of the four borders, and black bars across the borders between them
        side = 200
        for x0, y0 in ((4, 400), (W - side - 4, 400), (800, 4), (800, H - side - 4)):  # minDistanceToBorder = 3
            mid = int(rng.integers(0, 1000))
            _paste(img, mid, x0, y0, side)
            ids.add(mid)
        for x0, y0, x1, y1 in ((0, 0, 300, 40), (W - 40, 0, W, 300), (W - 300, H - 40, W, H), (0, H - 300, 40, H), (1300, 0, 1340, 200)):
            img[y0:y1, x0:x1] = 0
    elif kind == "length_min":
        # 1-pixel quadrilateral outlines whose outer contour has min_len - 1, min_len, min_len + 3 and min_len - 5 points: 4-gons, so
        # the length filter alone decides whether they are candidates
        ids = _four_markers(img, 320, W, H, rng, pad=0)
        n0 = min_len(W, H)
        for row, n in enumerate((n0 - 1, n0, n0 + 3, n0 - 5)):
            for k in range(6):
                _quad_outline(img, 20 + 48 * k, 20 + 110 * row, n)
    elif kind == "length_max":
        # zigzag closed 1-pixel curves of max_len - 1, max_len, max_len + 1 and max_len + 2 points
        n1 = max_len(W, H)
        for row, n in enumerate((n1 - 1, n1, n1 + 1, n1 + 2)):
            _zigzag(img, 10, 20 + 110 * row, n)
    elif kind == "segments":
        # horizontal 1-pixel segments of 66 pixels every second row, 1-pixel gaps between them; two markers in the top right corner
        for y in range(0, H, 2):
            for x in range(0, W - 66, 67):
                if not (x + 66 > W - 270 and y < 270):
                    img[y, x : x + 66] = 0
        for mid, (x0, y0) in zip(rng.choice(1000, 2, replace=False), ((W - 250, 20), (W - 125, 140))):
            _paste(img, int(mid), x0, y0, 100)
            ids.add(int(mid))
    elif kind == "lines":
        img[::2, :] = 0  # 1-pixel lines: every plane has H / 2 contours of 2 (W - 1) points
        img[:, 1500:] = 205
        ids = _four_markers(img, 1500, W, H, rng, pad=0)
        img[:, 1499] = 205
    return np.repeat(img[:, :, None], 3, axis=2), ids


@functools.lru_cache(maxsize=None)
def _quad_mask(n):
    """A 1-pixel outline of a quadrilateral (a rectangle with one slanted side, cv2.polylines) whose outer contour has exactly n
    points and approximates to a convex 4-gon (approxPolyDP at polygonalApproxAccuracyRate 0.01)."""
    for w in range(6, 60):
        for h in range(6, 60):
            for d in range(0, 6):
                m = np.zeros((h + 5, w + d + 5), np.uint8)
                cv2.polylines(m, [np.array([[2, 2], [2 + w, 2], [2 + w + d, 2 + h], [2, 2 + h]], np.int32)], True, 1, 1, cv2.LINE_8)
                cs, _ = cv2.findContours(m, cv2.RETR_EXTERNAL, cv2.CHAIN_APPROX_NONE)
                if len(cs) != 1 or len(cs[0]) != n:
                    continue
                ap = cv2.approxPolyDP(cs[0], 0.01 * n, True)
                if len(ap) == 4 and cv2.isContourConvex(ap):
                    return m.astype(bool)
    raise ValueError(n)


def _quad_outline(img, x0, y0, n):
    m = _quad_mask(n)
    img[y0 : y0 + m.shape[0], x0 : x0 + m.shape[1]][m] = 0


def _zigzag(img, x0, y0, n, w=600, h=60):
    """A closed 1-pixel curve whose outer contour has exactly n points: a w x h rectangle outline (2 (w - 1) + 2 (h - 1) points), with
    1-pixel teeth on its top edge (a tooth of height t adds 2 t - 2 points) and, for odd n, a chamfered corner (one point less)."""
    img[y0, x0 : x0 + w] = 0
    img[y0 + h - 1, x0 : x0 + w] = 0
    img[y0 : y0 + h, x0] = 0
    img[y0 : y0 + h, x0 + w - 1] = 0
    extra = n + n % 2 - (2 * (w - 1) + 2 * (h - 1))
    teeth, rest = divmod(extra, 16)  # teeth of height 9, then one of height rest / 2 + 1
    for k in range(teeth + 1):
        t = 9 if k < teeth else rest // 2 + 1
        img[y0 - t : y0, x0 + 3 + 3 * k] = 0
    if n % 2:
        img[y0 + h - 1, x0] = 205


@functools.lru_cache(maxsize=None)
def render(name):
    """(BGR frame, set of rendered marker ids)."""
    return _render(CASES[name])


# ---- start cracks counted on the CPU --------------------------------------------------------------------------------------------
def row_starts(plane):
    """halo_row_starts applied to a whole {0,1} plane laid out in 30-pixel halo tiles: (left, right) start masks.  The rules that look
    two columns away (L2, R2) do not apply in the first / last interior column of a tile, whose neighbours there lie outside the tile
    word."""
    P = np.zeros((plane.shape[0] + 2, plane.shape[1] + 4), bool)
    P[1:-1, 2:-2] = plane != 0
    H, W = plane.shape

    def at(dy, dx):
        return P[1 + dy : 1 + dy + H, 2 + dx : 2 + dx + W]

    mid, mid_l, mid_r, mid_l2, mid_r2 = at(0, 0), at(0, -1), at(0, 1), at(0, -2), at(0, 2)
    up, up_l, up_r, up_l2, up_r2 = at(-1, 0), at(-1, -1), at(-1, 1), at(-1, -2), at(-1, 2)
    dn, dn_l, dn_r = at(1, 0), at(1, -1), at(1, 1)
    col = (np.arange(W) % HALO_T + 1)[None, :]
    lone = mid & ~(up | up_l | up_r | mid_l | mid_r | dn | dn_l | dn_r)
    left = mid & ~mid_l & ~(up & ~up_l) & ~lone & ~(~up & ~up_l & up_r) & ~(up_l & ~mid_l2 & ~up_l2 & (col >= 2))
    right = mid & ~mid_r & ~(up & ~up_r) & ~lone & ~(~up & ~up_r & up_l) & ~(up_r & ~mid_r2 & ~up_r2 & (col <= HALO_T - 1))
    return left, right


def start_counts(planes):
    """[scales, 2] start cracks per plane and side."""
    out = np.zeros((len(planes), 2), np.int64)
    for s, p in enumerate(planes):
        left, right = row_starts(p)
        out[s] = left.sum(), right.sum()
    return out


def start_queue_cap(W, H, max_batch=1):
    """Entries per side of the start queue fid_create allocates."""
    return (6 * W * H * max_batch + 65536) // 2


def in_range_counts(planes, W, H):
    """(contours, points) with min_len <= n <= max_len over all planes, cv2.findContours (RETR_LIST, CHAIN_APPROX_NONE)."""
    lo, hi = min_len(W, H), max_len(W, H)
    nc = npt = 0
    for p in planes:
        cs, _ = cv2.findContours(p, cv2.RETR_LIST, cv2.CHAIN_APPROX_NONE)
        n = np.fromiter(map(len, cs), np.int64, len(cs))
        n = n[(n >= lo) & (n <= hi)]
        nc += len(n)
        npt += int(n.sum())
    return nc, npt


def contour_lengths(plane):
    """Lengths of every contour of a plane, cv2's list order."""
    cs, _ = cv2.findContours(plane, cv2.RETR_LIST, cv2.CHAIN_APPROX_NONE)
    return np.fromiter(map(len, cs), np.int64, len(cs))


# What each case is for, pinned on the CPU by tests/test_hostsim_contour_capacity.py:
#   queue   the start cracks of a one-frame chunk exceed the queue (3 per pixel and side): "over" or "fits"
#   chains  in-range contours past 65536: "over" or "fits"; points: in-range contour points past the handle's 4 W H + 65536
def expect(name):
    c = CASES[name]
    over_q = c["kind"] == "texture" and c["texture"] in ("checker1", "dither1")
    return dict(queue="over" if over_q else "fits", chains="over" if c["kind"] == "segments" else "fits",
                points="over" if c["kind"] == "lines" else "fits")
