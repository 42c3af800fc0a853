"""The C++ node glue's localization (FiducialSlam::localize and publishedPose in fiducials_b200/csrc/node_glue.hpp): it builds and
links without a GPU; on a GPU it localizes one /fiducial_vertices message against a map file and prints what the Python
FiducialSlam computes from the same map and corners."""
import os
import subprocess

import numpy as np
import pytest

import map_ba_cases as mc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MOUNT = [0.12, -0.03, 0.35, 0.5, -0.5, 0.5, 0.5]


def _build(exe):
    from test_node_glue import _build as build_lib  # builds the library if needed

    build_lib()
    libdir = os.path.join(ROOT, "fiducials_b200")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "node_glue_localize_main.cpp"), "-L" + libdir, "-lfiducials_b200",
                           "-Wl,-rpath," + libdir, "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64", "-lcudart"])


def test_builds_and_links(tmp_path):
    exe = str(tmp_path / "node_glue_localize_main")
    _build(exe)
    assert os.access(exe, os.X_OK)


@pytest.mark.gpu
def test_one_frame_matches_the_python_node(tmp_path):
    from fiducials_b200.node import FiducialSlam

    exe = str(tmp_path / "node_glue_localize_main")
    _build(exe)
    sc = mc.make_scene(3, dist=True, noise=0.5, n_frames=8)
    rows = mc.file_entries(sc)
    with open(tmp_path / "map.txt", "w") as fp:
        for r in rows:
            fp.write("%d %s %d\n" % (r[0], " ".join(repr(float(v)) for v in r[1:8]), r[8]))
    f = int(np.argmax(sc["counts"]))
    n = int(sc["counts"][f])
    with open(tmp_path / "vertices.txt", "w") as fp:
        for j in range(n):
            fp.write("%d %s\n" % (sc["fids"][f, j], " ".join("%.9g" % v for v in sc["corners"][f, j].ravel())))
    K, D = sc["K"], sc["D"]
    args = [exe, str(tmp_path / "map.txt"), str(tmp_path / "vertices.txt")] + [repr(float(v)) for v in (K[0, 0], K[1, 1], K[0, 2], K[1, 2])] + \
        [repr(float(v)) for v in D] + [repr(float(sc["fiducial_len"]))]
    r = subprocess.run(args, capture_output=True, text=True, check=True)
    L = [l.split() for l in r.stdout.splitlines() if l.startswith("L ")][0]
    P = [np.array(l.split()[1:], float) for l in r.stdout.splitlines() if l.startswith("P ")]
    slam = FiducialSlam(max_fiducials=64)
    slam.loadMapFile(str(tmp_path / "map.txt"))
    loc = slam.localize(sc["counts"][f:f + 1], sc["fids"][f:f + 1, :n], sc["corners"][f:f + 1, :n], K, D, sc["fiducial_len"], T_camBase=MOUNT)[0]
    assert [int(v) for v in L[1:5]] == [1, n, int(loc["start"]), 1] and loc["status"] == 1
    vals = np.array(L[5:], float)
    assert np.array_equal(vals, np.r_[loc["t"], loc["q"], loc["object_error"], loc["covariance"]])
    robot = type("R", (), dict(t=[1.0, 2.0, 0.5], q=[0.0, 0.0, 0.0, 1.0], variance=0.25))()
    for thr, got in zip((-1.0, 1e9), P):
        slam.multi_error_threshold = thr
        t, q, cov = slam.published_pose(robot, loc)
        assert np.array_equal(got, np.r_[t, q, cov])
