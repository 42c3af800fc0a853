"""Cost of fid_map_localize (DESIGN.md f17, §4): a C5-style ceiling map of 500 entries (tests/map_ba_cases.make_scene, 1 m pitch,
its fold-perturbed start map) loaded with fid_map_load, and batches of 128 and 4 096 frames of seeded projected corners (about 10
markers per frame, 0.5 px noise, plumb_bob distortion).  Per batch size: the call's time by a host clock around the synchronous
call (it ends in a stream synchronise), after warm-up calls of the same shape, and frames/s.  The GPU's name and power limit are
read in the same run.  Usage: python tools/bench_map_localize.py [--reps 20]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import map_ba_cases as mc  # noqa: E402
from fiducials_b200.node import FiducialSlam  # noqa: E402


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
        return q.stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    # 1 024 distinct frames along the lawn-mower path; the 4 096-frame batch repeats them four times (the same work per frame)
    sc = mc.make_scene(5, n_markers=500, n_frames=1024, visible=10, noise=0.5, dist=True)
    slam = FiducialSlam(max_fiducials=512)
    slam.loadMap(mc.file_entries(sc))
    print("gpu: %s" % gpu_info())
    for n in (128, 4096):
        idx = np.arange(n) % len(sc["counts"])
        counts, fids, corners = sc["counts"][idx], sc["fids"][idx], sc["corners"][idx]
        for _ in range(args.warmup):
            out = slam.localize(counts, fids, corners, sc["K"], sc["D"], sc["fiducial_len"])
        ts = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            out = slam.localize(counts, fids, corners, sc["K"], sc["D"], sc["fiducial_len"])
            ts.append(time.perf_counter() - t0)
        ms = 1e3 * float(np.median(ts))
        print(json.dumps(dict(frames=n, markers_per_frame=round(float(np.mean(counts)), 2), posed=int(np.sum(out["status"] == 1)), median_ms=round(ms, 3),
                              min_ms=round(1e3 * min(ts), 3), max_ms=round(1e3 * max(ts), 3), frames_per_s=round(n / (ms / 1e3), 1),
                              mean_lm_iters=round(float(np.mean(out["lm_iters"])), 2))))


if __name__ == "__main__":
    main()
