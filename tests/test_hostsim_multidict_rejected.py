"""What cv2 4.13's detectMarkersMultiDict returns as rejectedImgPoints (DESIGN.md finding 15): why the library does not return it.  The
checks run cv2 alone, on 1080p frames with markers of four families; they back the finding's claims, and fail if a later OpenCV
changes the rule.  CPU only."""
import cv2
import numpy as np

import multidict_oracle as mo

A = mo.A
DL = mo.DICT_LISTS["four"]


def _frame(seed):
    """28 axis-aligned markers of the four families in a 7 x 4 grid, one perspective warp, noise."""
    rng = np.random.default_rng(seed)
    D = [A.getPredefinedDictionary(d) for d in DL]
    img = np.full((1080, 1920), 200, np.uint8)
    for k in range(28):
        gy, gx = divmod(k, 7)
        s = int(rng.integers(60, 200))
        m = np.rot90(A.generateImageMarker(D[k % 4], int(rng.integers(0, 50)), s, borderBits=1), int(rng.integers(4)))
        img[40 + gy * 260:40 + gy * 260 + s, 40 + gx * 260:40 + gx * 260 + s] = m
    img = cv2.warpPerspective(img, np.array([[1, 0.05, 0], [0.02, 1, 0], [1e-5, 2e-5, 1]]), (1920, 1080), borderValue=200)
    return np.clip(img + rng.normal(0, 3, img.shape), 0, 255).astype(np.uint8)


def _key(q):
    """The squared distance of the quad's centroid from the origin, in float32."""
    q = np.asarray(q, np.float32).reshape(4, 2)
    ax = np.float32(np.float32(np.float32(q[0, 0] + q[1, 0]) + q[2, 0]) + q[3, 0]) * np.float32(0.25)
    ay = np.float32(np.float32(np.float32(q[0, 1] + q[1, 1]) + q[2, 1]) + q[3, 1]) * np.float32(0.25)
    return float(np.float32(ax * ax + ay * ay))


def _t(q):
    return tuple(np.asarray(q, np.float32).ravel().tolist())


def test_rejected_list_rule():
    not_intersection = duplicates = outside_union = 0
    for seed in range(3):
        img = _frame(seed)
        bgr = cv2.cvtColor(img, cv2.COLOR_GRAY2BGR)
        for method in (0, 1):
            _, _, _, rej = mo.cv2_multi(bgr, DL, method)
            singles = [set(map(_t, mo.cv2_single(bgr, d, method)[2])) for d in DL]
            got = list(map(_t, rej))
            keys = [_key(q) for q in got]
            assert keys == sorted(keys), (seed, method)  # sorted by the centroid's squared distance from the origin
            inter, union = set.intersection(*singles), set.union(*singles)
            not_intersection += set(got) != inter
            duplicates += len(got) != len(set(got))
            if method == 0:
                assert set(got) <= union, seed  # without refinement, every quad is rejected by some single run
            else:
                outside_union += len(set(got) - union) > 0
    assert not_intersection == 6  # never the intersection of the single runs
    assert duplicates >= 3  # duplicate quads are kept
    assert outside_union >= 1  # under SUBPIX it holds quads no single run rejects
