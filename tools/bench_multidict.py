"""Cost of detecting several dictionaries in one pass (fid_set_dictionaries) on one GPU.

The workload is a 64-frame batch of rendered 1080p frames in device memory with markers of two or three families (20 markers per
frame, random family, id, size and quarter turn, a mild perspective warp, blur and noise), run in chunks of 32 through the
submit/collect loop with two batches in flight (as bench.py runs it), with a camera.  For each family set it compares
  (a) one handle with the N dictionaries,
  (b) N single-dictionary handles over the same frames (each batch submitted to every handle),
  (c) the first dictionary alone on one handle,
in frames/s (alternating runs) and, from a torch.profiler run of its own, the device time per 64-frame batch of each kernel.

Prints the card name and power limit read in the same run; --out DIR also writes the numbers as JSON.
    python tools/bench_multidict.py [--steps 6] [--runs 3] [--out DIR]"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

from bench_marker_refine import card
from fiducials_b200 import synth
from fiducials_b200.node import Detector, default_params
import multidict_oracle as mo

W, H, N, CHUNK = 1920, 1080, 64, 32  # 32-frame chunks (three 1080p handles of 64-frame chunks do not fit in 80 GB), two per batch
A = mo.A
FAMILIES = {"two": [A.DICT_5X5_1000, A.DICT_APRILTAG_36h11], "three": [A.DICT_5X5_1000, A.DICT_APRILTAG_36h11, A.DICT_6X6_250]}
KERNELS = ("k_threshold", "k_walk", "k_emit", "k_approx", "k_sort_group", "k_identify_first", "k_identify_retry", "k_contour_refine", "k_finish", "k_dict_merge")


def handles(dl, mode):
    if mode == "a":
        d = Detector(default_params(dictionary=dl[0]), 0, W, H, CHUNK)
        d.set_dictionaries([(x, 0, 0.0) for x in dl])
        return [d]
    if mode == "b":
        return [Detector(default_params(dictionary=x), 0, W, H, CHUNK) for x in dl]
    return [Detector(default_params(dictionary=dl[0]), 0, W, H, CHUNK)]


def loop(dets, dev, K, steps):
    """submit/collect with two batches in flight per handle; frames/s (frames of the stream, every handle run on each) over
    `steps` batches after the queue is primed; the markers per batch."""
    args = (K, np.zeros(5), 0.14)
    kw = dict(on_device=True, n_frames=N, width=W, height=H)
    outs = [None] * len(dets)
    for d in dets:
        d.submit_batch(dev.data_ptr(), *args, **kw)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        for i, d in enumerate(dets):
            d.submit_batch(dev.data_ptr(), *args, **kw)
            outs[i] = d.collect_batch(outs[i])
    for i, d in enumerate(dets):
        outs[i] = d.collect_batch(outs[i])
    fps = N * (steps + 1) / (time.perf_counter() - t0)
    return fps, sum(int(o[0].sum()) for o in outs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: nothing to measure")
    K, _ = synth.camera_for(W, H)
    res = {"card": card(), "frames_per_batch": N, "chunk": CHUNK, "sets": {}}
    for name, dl in FAMILIES.items():
        frames = [mo.render_mixed(W, H, dl, 500 + i, n_markers=20) for i in range(16)]
        dev = torch.from_numpy(np.ascontiguousarray(np.stack([frames[i % 16] for i in range(N)]))).cuda()
        r = {"dictionaries": dl, "device_ms_per_batch": {}, "markers_per_batch": {}, "frames_per_s": {m: [] for m in "abc"}}
        for m in "abc":  # the handles of one configuration at a time
            dets = handles(dl, m)
            loop(dets, dev, K, 1)  # warm-up
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                _, n_markers = loop(dets, dev, K, 1)  # two batches per handle
                torch.cuda.synchronize()
            r["device_ms_per_batch"][m] = {k: round(sum(e.device_time for e in prof.events() if k + "(" in e.name or k + "<" in e.name) / 1000.0 / 2, 3)
                                           for k in KERNELS}
            r["markers_per_batch"][m] = n_markers // 2
            for d in dets:
                d.close()
        for _ in range(args.runs):  # alternating runs, each on handles of its own
            for m in "abc":
                dets = handles(dl, m)
                loop(dets, dev, K, 1)
                r["frames_per_s"][m].append(round(loop(dets, dev, K, args.steps)[0], 1))
                for d in dets:
                    d.close()
        r["median_frames_per_s"] = {m: float(np.median(v)) for m, v in r["frames_per_s"].items()}
        res["sets"][name] = r
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_multidict.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
