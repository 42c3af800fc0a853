"""FiducialsNode with several dictionaries (Python and the C++ node glue): the per-frame path (imageCallback -> poseEstimateCallback, one
fid_pose per dictionary on published ids) gives the messages of the batch path (process_batch), ignore_fiducials and
fiducial_len_override are keyed by published id, and FiducialSlam fed the node's messages keeps two families with equal raw ids apart."""
import os
import subprocess

import numpy as np
import pytest

from fiducials_b200 import synth
from fiducials_b200.node import FiducialSlam, FiducialsNode
import multidict_oracle as mo

pytestmark = pytest.mark.gpu
A = mo.A
W, H = 1280, 720
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D0 = A.DICT_6X6_250
EXTRA = [(A.DICT_APRILTAG_36h11, 1000, 0.2), (A.DICT_4X4_50, 2000, 0.0)]
DL = [D0] + [e[0] for e in EXTRA]


def _node(**kw):
    node = FiducialsNode(dictionary=D0, fiducial_len=0.14, max_width=W, max_height=H, max_batch=4, dictionaries=EXTRA, **kw)
    K, D = synth.camera_for(W, H)
    node.camInfoCallback(K, D, "camera")
    return node


def _frames(n, seed):
    return [mo.render_mixed(W, H, DL, seed + i, n_markers=12) for i in range(n)]


def _key(t):
    return (t.fiducial_id, t.transform.translation, t.transform.rotation, t.image_error, t.object_error, t.fiducial_area)


def test_per_frame_equals_batch():
    frames = _frames(3, 300)
    first = frames[0]
    ids0, _, di0 = mo.host_multi(first, DL, 1)
    pub0 = ids0 + np.array([0, 1000, 2000])[di0]
    ignore = int(pub0[di0 == 1][0]) if (di0 == 1).any() else 1
    override = {int(pub0[di0 == 2][0]) if (di0 == 2).any() else 2: 0.33}
    per_frame = _node(ignore_fiducials=[ignore], fiducial_len_override=override)
    batch = _node(ignore_fiducials=[ignore], fiducial_len_override=override)
    msgs = batch.process_batch(np.stack(frames))
    n_families = set()
    for f, bgr in enumerate(frames):
        fva = per_frame.imageCallback(bgr)
        fta = per_frame.poseEstimateCallback(fva)
        ids, corners, di = mo.host_multi(bgr, DL, 1)
        pub = ids + np.array([0, 1000, 2000])[di]
        keep = pub != ignore
        assert [v.fiducial_id for v in fva.fiducials] == pub[keep].tolist()
        got_c = np.array([[v.x0, v.y0, v.x1, v.y1, v.x2, v.y2, v.x3, v.y3] for v in fva.fiducials], np.float32).reshape(-1, 4, 2)
        assert np.array_equal(got_c, corners[keep])
        assert [_key(t) for t in fta.transforms] == [_key(t) for t in msgs[f].transforms]
        n_families |= set(di.tolist())
    assert n_families == {0, 1, 2}
    assert ignore not in [t.fiducial_id for m in msgs for t in m.transforms]


def test_slam_keeps_families_apart():
    g = np.full((H, W), 200, np.uint8)
    g[200:460, 200:460] = A.generateImageMarker(A.getPredefinedDictionary(D0), 5, 260, borderBits=1)
    g[200:460, 800:1060] = A.generateImageMarker(A.getPredefinedDictionary(EXTRA[0][0]), 5, 260, borderBits=1)
    bgr = np.ascontiguousarray(np.repeat(g[:, :, None], 3, axis=2))
    node = _node()
    fta = node.poseEstimateCallback(node.imageCallback(bgr))
    assert sorted(t.fiducial_id for t in fta.transforms) == [5, 1005]
    slam = FiducialSlam()
    ident = [0, 0, 0, 0, 0, 0, 1]
    for _ in range(13):
        slam.transformCallback(fta, ident, ident)
    assert sorted(int(e.fiducial_id) for e in slam.entries()) == [5, 1005]


def test_node_glue_matches_python_node(tmp_path):
    from test_node_glue import _build  # builds the library if needed

    _build()
    exe = str(tmp_path / "node_glue_multidict_main")
    libdir = os.path.join(ROOT, "fiducials_b200")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "node_glue_multidict_main.cpp"), "-L" + libdir, "-lfiducials_b200",
                           "-Wl,-rpath," + libdir, "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64", "-lcudart"])
    bgr = _frames(1, 400)[0]
    ids, _, di = mo.host_multi(bgr, DL, 1)
    pub = ids + np.array([0, 1000, 2000])[di]
    ignore, override = int(pub[0]), int(pub[-1])
    raw = tmp_path / "f.bgr"
    raw.write_bytes(bgr.tobytes())
    args = [exe, str(raw), str(W), str(H), str(D0), "0.14", str(ignore), str(override), "0.3"] + [str(v) for e in EXTRA for v in e]
    r = subprocess.run(args, capture_output=True, text=True, check=True)
    node = FiducialsNode(dictionary=D0, fiducial_len=0.14, max_width=W, max_height=H, dictionaries=EXTRA, ignore_fiducials=[ignore],
                         fiducial_len_override={override: 0.3})
    K = np.array([[0.73 * W, 0, W / 2.0], [0, 0.73 * W, H / 2.0], [0, 0, 1]])
    node.camInfoCallback(K, [-0.2, 0.05, 0.001, -0.001, 0.0], "camera")
    fva = node.imageCallback(bgr)
    fta = node.poseEstimateCallback(fva)
    V = [l.split() for l in r.stdout.splitlines() if l.startswith("V ")]
    T = [l.split() for l in r.stdout.splitlines() if l.startswith("T ")]
    assert [int(v[1]) for v in V] == [v.fiducial_id for v in fva.fiducials] and ignore not in [int(v[1]) for v in V]
    assert len(T) == len(fta.transforms) > 3
    for t, m in zip(T, fta.transforms):
        assert int(t[1]) == m.fiducial_id
        vals = [float(x) for x in t[2:]]
        assert vals == list(m.transform.translation) + list(m.transform.rotation) + [m.image_error, m.object_error, m.fiducial_area]
