"""Cost of the ChArUco diamond stage of the batch calls (fid_set_diamonds) on one GPU.

The workload is a 128-frame batch of rendered 1080p frames in device memory, each with 8 diamonds (4 x 2, random ids, in-plane
turns and tilts, blurred), run in chunks of 64 through the submit/collect loop with two batches in flight (as bench.py runs it),
with a camera.  It reports the device time of k_diamond per 128-frame batch (torch.profiler, a run of its own), the diamonds found
per batch, then frames/s with diamonds off and on on the same handle, in alternating runs.

Prints the card name and power limit read in the same run; --out DIR also writes the numbers as JSON.
    python tools/bench_diamond.py [--steps 10] [--runs 3] [--out DIR]"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import cv2
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

from bench_marker_refine import card
from fiducials_b200 import synth
from fiducials_b200.node import Detector, default_params
import charuco_oracle as co
import diamond_oracle as do

W, H, N, CHUNK = 1920, 1080, 128, 64
SQUARE, MARKER = 0.04, 0.03
KERNELS = ("k_diamond", "k_finish")


def rendered_frames(K, n_distinct=16, seed=0):
    """n_distinct frames of 8 diamonds each, repeated to N frames (BGR)."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n_distinct):
        g = np.full((H, W), 128, np.uint8)
        ids = rng.permutation(250)
        for k in range(8):
            centre = (W * (k % 4 + 0.5) / 4, H * (k // 4 + 0.5) / 2)
            R, t = do.diamond_pose(rng, K, W, H, SQUARE, "far", centre, int(rng.integers(4)))
            do.render_diamond(g, ids[4 * k:4 * k + 4], SQUARE, MARKER, R, t, K)
        out.append(cv2.cvtColor(co.blur_noise(g, rng, True, 0.3), cv2.COLOR_GRAY2BGR))
    return np.ascontiguousarray(np.stack([out[i % n_distinct] for i in range(N)]))


def loop(det, dev, K, steps):
    """submit/collect with two batches in flight; frames/s over `steps` batches after the queue is primed."""
    args = (K, np.zeros(5), 0.14)
    kw = dict(on_device=True, n_frames=N, width=W, height=H)
    out = None
    det.submit_batch(dev.data_ptr(), *args, **kw)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        det.submit_batch(dev.data_ptr(), *args, **kw)
        out = det.collect_batch(out)
    out = det.collect_batch(out)
    return N * (steps + 1) / (time.perf_counter() - t0), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: nothing to measure")
    K, _ = synth.camera_for(W, H)
    frames = rendered_frames(K)
    dev = torch.from_numpy(frames).cuda()
    det = Detector(default_params(dictionary=do.DICT_ID), 0, W, H, CHUNK)
    det.set_diamonds(SQUARE, MARKER)
    loop(det, dev, K, 2)  # warm-up
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        loop(det, dev, K, 1)  # two batches
        torch.cuda.synchronize()
    dev_ms = {k: sum(e.device_time for e in prof.events() if k + "(" in e.name) / 1000.0 / 2 for k in KERNELS}
    found = sum(len(d[0]) for d in det.last_diamonds())
    fps = {"off": [], "on": []}
    for _ in range(args.runs):
        for mode in ("off", "on"):
            det.set_diamonds(SQUARE if mode == "on" else None, MARKER)
            loop(det, dev, K, 1)
            fps[mode].append(round(loop(det, dev, K, args.steps)[0], 1))
    det.close()
    res = {"card": card(), "frames_per_batch": N, "chunk": CHUNK, "diamonds_per_batch": found, "device_ms_per_batch": dev_ms, "frames_per_s": fps,
           "median_off": float(np.median(fps["off"])), "median_on": float(np.median(fps["on"]))}
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_diamond.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
