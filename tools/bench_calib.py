"""Device time of fid_calibrate_camera (CUDA events around its device work, median of --reps runs after a warm-up) for 100 / 400 /
1 000 / 4 000 views of a 7x5 and a 12x9 ChArUco board (24 and 88 corners per view, 30 % of the views partly covered), beside
the wall time of cv2.calibrateCamera on this host's CPU for the sizes up to --cv2-max views.  Prints one JSON line (and writes it
to --out) with the card's name and power limit, read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import calib_cases as cc  # noqa: E402
from fiducials_b200 import _lib, calib  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return q.strip().splitlines()[0]
    except Exception as e:  # the numbers below still come from the device events
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", default="100,400,1000,4000")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cv2-max", type=int, default=100)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "cpu_threads": os.cpu_count(), "cv2": cv2.__version__, "rows": []}
    for name, grid in (("7x5", (6, 4)), ("12x9", (11, 8))):
        for nv in [int(v) for v in a.views.split(",")]:
            O, I, K, D = cc.make_problem(7 + nv, nv, grid, (1920, 1080), "mild", 0.2, 0.3)
            st = _lib.fid_calib_stats()
            r = calib.calibrate_camera(O, I, (1920, 1080), stats=st)  # warm-up (module load)
            ms, wall = [], []
            for _ in range(a.reps):
                t0 = time.perf_counter()
                r = calib.calibrate_camera(O, I, (1920, 1080), stats=st)
                wall.append((time.perf_counter() - t0) * 1e3)
                ms.append(st.device_ms)
            row = {"board": name, "views": nv, "points": int(sum(len(o) for o in O)), "device_ms": float(np.median(ms)), "call_ms": float(np.median(wall)),
                   "steps": int(st.n_steps), "launches": int(st.kernel_launches),
                   "rms": float(r[0])}
            if nv <= a.cv2_max:
                t0 = time.perf_counter()
                ref = cv2.calibrateCamera(O, I, (1920, 1080), None, None)
                row["cv2_s"] = time.perf_counter() - t0
                row["rms_rel_vs_cv2"] = float(r[0] / ref[0] - 1)
            res["rows"].append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
