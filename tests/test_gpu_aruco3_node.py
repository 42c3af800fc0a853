"""FiducialsNode with detection on a downscaled frame (Python `aruco3=` and the C++ node glue's setAruco3): the messages carry the
markers of the mode (ids and full-resolution corners of the host chain, tests/hostsim/aruco3_hostsim.cpp), the per-frame path
(imageCallback -> poseEstimateCallback) gives the messages of the batch path (process_batch), and the C++ glue prints what the Python
node publishes."""
import os
import subprocess

import numpy as np
import pytest

from fiducials_b200 import synth
from fiducials_b200.node import FiducialsNode
import aruco3_oracle as a3

pytestmark = pytest.mark.gpu
A = a3.A
W, H = 1920, 1080
D0 = A.DICT_6X6_250
RATIO, MIN_SIDE = 0.02, 32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _frames(n, seed):
    return [a3.render(W, H, D0, seed + i, 12, side_range=(0.2, 0.8)) for i in range(n)]


def _key(t):
    return (t.fiducial_id, t.transform.translation, t.transform.rotation, t.image_error, t.object_error, t.fiducial_area)


def test_per_frame_equals_batch():
    frames = _frames(3, 800)
    K, D = synth.camera_for(W, H)
    per_frame = FiducialsNode(dictionary=D0, fiducial_len=0.14, max_width=W, max_height=H, aruco3=(RATIO, MIN_SIDE))
    batch = FiducialsNode(dictionary=D0, fiducial_len=0.14, max_width=W, max_height=H, max_batch=4, aruco3=(RATIO, MIN_SIDE))
    for node in (per_frame, batch):
        node.camInfoCallback(K, D, "camera")
    msgs = batch.process_batch(np.stack(frames))
    n = 0
    for f, bgr in enumerate(frames):
        fva = per_frame.imageCallback(bgr)
        fta = per_frame.poseEstimateCallback(fva)
        ids, corners = a3.host_detect(bgr, D0, MIN_SIDE, RATIO)
        assert [v.fiducial_id for v in fva.fiducials] == ids.tolist()
        got_c = np.array([[v.x0, v.y0, v.x1, v.y1, v.x2, v.y2, v.x3, v.y3] for v in fva.fiducials], np.float32).reshape(-1, 4, 2)
        assert np.array_equal(got_c, corners)
        assert [_key(t) for t in fta.transforms] == [_key(t) for t in msgs[f].transforms]
        n += len(fta.transforms)
    assert n >= 10


def test_node_glue_matches_python_node(tmp_path):
    from test_node_glue import _build  # builds the library if needed

    _build()
    exe = str(tmp_path / "node_glue_aruco3_main")
    libdir = os.path.join(ROOT, "fiducials_b200")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "node_glue_aruco3_main.cpp"), "-L" + libdir, "-lfiducials_b200",
                           "-Wl,-rpath," + libdir, "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64", "-lcudart"])
    bgr = _frames(1, 900)[0]
    raw = tmp_path / "f.bgr"
    raw.write_bytes(bgr.tobytes())
    r = subprocess.run([exe, str(raw), str(W), str(H), str(D0), "0.14", str(RATIO), str(MIN_SIDE)], capture_output=True, text=True, check=True)
    node = FiducialsNode(dictionary=D0, fiducial_len=0.14, max_width=W, max_height=H, aruco3=(RATIO, MIN_SIDE))
    K = np.array([[0.73 * W, 0, W / 2.0], [0, 0.73 * W, H / 2.0], [0, 0, 1]])
    node.camInfoCallback(K, [-0.2, 0.05, 0.001, -0.001, 0.0], "camera")
    fva = node.imageCallback(bgr)
    fta = node.poseEstimateCallback(fva)
    ids, corners = a3.host_detect(bgr, D0, MIN_SIDE, RATIO)
    V = [l.split() for l in r.stdout.splitlines() if l.startswith("V ")]
    T = [l.split() for l in r.stdout.splitlines() if l.startswith("T ")]
    assert [int(v[1]) for v in V] == [v.fiducial_id for v in fva.fiducials] == ids.tolist()
    assert np.array_equal(np.array([[float(x) for x in v[2:]] for v in V], np.float32).reshape(-1, 4, 2), corners)
    assert len(T) == len(fta.transforms) > 3
    for t, m in zip(T, fta.transforms):
        assert int(t[1]) == m.fiducial_id
        vals = [float(x) for x in t[2:]]
        assert vals == list(m.transform.translation) + list(m.transform.rotation) + [m.image_error, m.object_error, m.fiducial_area]
