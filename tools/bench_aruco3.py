"""Cost and yield of useAruco3Detection (fid_set_aruco3) on one GPU.

The workloads are the C2 (1080p) and C4 (4K) frame streams of synth.make_config_stream, in device memory, run through the
submit/collect loop with two batches in flight (as bench.py runs it), with a camera.  For each workload it compares the mode off
and on at minMarkerLengthRatioOriginalImg 0.02 and 0.05 (minSideLengthCanonicalImg 32):
  - frames/s, medians of alternating runs with their spread;
  - markers found per frame: the mode drops markers below the minimum side by design, so a rate means nothing without it;
  - from a torch.profiler run of its own, the device time per batch of the new kernels (planes, identification on the pyramid,
    the corner stage) and of the front-end kernels they shrink.
Prints the card name and power limit read in the same run; --out DIR also writes the numbers as JSON.
    python tools/bench_aruco3.py [--steps 6] [--runs 3] [--out DIR]"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

from bench_marker_refine import card
from fiducials_b200 import synth
from fiducials_b200.node import Detector, default_params

WORKLOADS = {"C2": 64, "C4": 16}  # frames per batch (C4: 4K frames, a quarter of the chunk)
SETTINGS = {"off": None, "r0.02": 0.02, "r0.05": 0.05}
KERNELS = ("k_gray", "k_a3_pyr_down", "k_a3_resize", "k_threshold", "k_walk", "k_emit", "k_approx", "k_sort_group", "k_identify_first", "k_identify_retry",
           "k_finish", "k_a3_corners", "k_recovered_pose")


def handle(W, H, n, d, ratio):
    det = Detector(default_params(dictionary=d), 0, W, H, n)
    if ratio is not None:
        det.set_aruco3(32, ratio)
    return det


def loop(det, dev, n, W, H, K, D, steps):
    kw = dict(on_device=True, n_frames=n, width=W, height=H)
    out = None
    det.submit_batch(dev.data_ptr(), K, D, 0.14, **kw)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    markers = 0
    for _ in range(steps):
        det.submit_batch(dev.data_ptr(), K, D, 0.14, **kw)
        out = det.collect_batch(out)
        markers += int(out[0].sum())
    out = det.collect_batch(out)
    return n * (steps + 1) / (time.perf_counter() - t0), markers / (n * steps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: nothing to measure")
    res = {"card": card(), "workloads": {}}
    for wl, n in WORKLOADS.items():
        frames, _, K, D, d = synth.make_config_stream(wl, n, seed=3)
        H, W = frames.shape[1:3]
        dev = torch.from_numpy(np.ascontiguousarray(frames)).cuda()
        r = {"frames_per_batch": n, "frames_per_s": {s: [] for s in SETTINGS}, "markers_per_frame": {}, "device_ms_per_batch": {}}
        for s, ratio in SETTINGS.items():
            det = handle(W, H, n, d, ratio)
            loop(det, dev, n, W, H, K, D, 1)  # warm-up
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                loop(det, dev, n, W, H, K, D, 1)  # two batches
                torch.cuda.synchronize()
            r["device_ms_per_batch"][s] = {k: round(sum(e.device_time for e in prof.events() if k + "(" in e.name or k + "<" in e.name) / 1000.0 / 2, 3)
                                           for k in KERNELS}
            r["markers_per_frame"][s] = round(loop(det, dev, n, W, H, K, D, 2)[1], 2)
            det.close()
        for _ in range(args.runs):  # alternating runs, each on a handle of its own
            for s, ratio in SETTINGS.items():
                det = handle(W, H, n, d, ratio)
                loop(det, dev, n, W, H, K, D, 1)
                r["frames_per_s"][s].append(round(loop(det, dev, n, W, H, K, D, args.steps)[0], 1))
                det.close()
        r["median_frames_per_s"] = {s: float(np.median(v)) for s, v in r["frames_per_s"].items()}
        r["spread_frames_per_s"] = {s: float(max(v) - min(v)) for s, v in r["frames_per_s"].items()}
        res["workloads"][wl] = r
        del dev
        torch.cuda.empty_cache()
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_aruco3.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
