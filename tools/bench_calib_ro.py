"""Device time of fid_calibrate_camera_ro (CUDA events around its device work, median of --reps runs after a warm-up) for printed
boards of 24, 88, 352 and 1 024 points x 30 / 100 / 1 000 views, beside the wall time of cv2.calibrateCameraROExtended on this
host's CPU where its dense solve is cheap enough (6 views + 3 points <= --cv2-max-params), and the achieved FP64 rate of the
dense kernels together (the SYRK of the views' Z and the blocked Cholesky: k_dense_syrk, k_dense_potrf, k_dense_trsm), from one
torch.profiler run per size with the FLOPs computed here from the shapes.  Prints one JSON line (and writes it to --out) with
the card's name and power limit, read in the same run."""
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
import calib_ro_cases as rc  # noqa: E402
from fiducials_b200 import _lib, calib  # noqa: E402

GRIDS = {24: (6, 4), 88: (11, 8), 352: (22, 16), 1024: (32, 32)}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return q.strip().splitlines()[0]
    except Exception as e:  # the numbers below still come from the device events
        return "unknown (%s)" % e


def dense_flops(n, nv, steps):
    """FP64 FLOPs of the SYRK of the views' Z (lower 32x32 tiles, K = 6 views) and of the blocked Cholesky, per computed system
    (steps taken + the final one), as the kernels compute them (a diagonal tile in full)."""
    mp = (9 + 3 * n + 31) // 32 * 32
    t = mp // 32
    syrk = t * (t + 1) // 2 * 32 * 32 * 2 * 6 * nv
    chol = 0
    for j in range(t):
        r = t - j - 1
        chol += 32 ** 3 // 3 + r * 32 * 32 * 32 + r * (r + 1) // 2 * 32 * 32 * 2 * 32
    return syrk * (steps + 1), chol * (steps + 1)


def kernel_ms(fn):
    """Device time of the dense kernels in one call of fn, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ms = 0.0
    for e in prof.events():
        if "k_dense_syrk" in e.name or "k_dense_potrf" in e.name or "k_dense_trsm" in e.name:
            ms += e.device_time / 1e3
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", default="24,88,352,1024")
    ap.add_argument("--views", default="30,100,1000")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cv2-max-params", type=int, default=1000)
    ap.add_argument("--profile", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "cpu_threads": os.cpu_count(), "cv2": cv2.__version__, "rows": []}
    for n in [int(p) for p in a.points.split(",")]:
        grid = GRIDS[n]
        for nv in [int(v) for v in a.views.split(",")]:
            O, I, K, D, _ = rc.make_printed_problem(5 + n + nv, nv, grid, (3840, 2160), "mild", 0.2, (1.004, 1.0), square=0.32 / max(grid))
            fixed = grid[0] - 1
            st = _lib.fid_calib_stats()
            run = lambda: calib.calibrate_camera_ro(O, I, (3840, 2160), fixed, stats=st)
            r = run()  # warm-up (module load)
            ms, wall = [], []
            for _ in range(a.reps):
                t0 = time.perf_counter()
                r = run()
                wall.append((time.perf_counter() - t0) * 1e3)
                ms.append(st.device_ms)
            row = {"points": n, "views": nv, "device_ms": float(np.median(ms)), "call_ms": float(np.median(wall)), "steps": int(st.n_steps),
                   "launches": int(st.kernel_launches), "rms": float(r[0])}
            if a.profile:
                # the Cholesky's trailing updates are k_dense_syrk launches too, so the kernels are timed together
                syrk_f, chol_f = dense_flops(n, nv, int(st.n_steps))
                row["dense_ms"] = kernel_ms(run)
                row["dense_gflop"] = (syrk_f + chol_f) / 1e9
                row["dense_tflops"] = (syrk_f + chol_f) / (row["dense_ms"] * 1e-3) / 1e12 if row["dense_ms"] else None
            if 6 * nv + 3 * n <= a.cv2_max_params:
                t0 = time.perf_counter()
                ref = rc.cv2_calibrate_ro(O, I, (3840, 2160), fixed)
                row["cv2_s"] = time.perf_counter() - t0
                row["rms_rel_vs_cv2"] = float(r[0] / ref["rms"] - 1)
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
