"""Cost of the board stages on a multi-dictionary handle (fid_set_family_boards / fid_set_family_charuco_boards) on one GPU.

The workload is a 64-frame batch of rendered 1080p frames in device memory with two families (DICT_5X5_1000 and AprilTag 36h11),
each with one 2 x 2 GridBoard (ids 0..3) and one 5 x 4 ChArUco board (ids 0..9), so every raw id is on the frame twice, under a
mild perspective warp, blur and noise.  It runs in chunks of 32 through the submit/collect loop with two batches in flight (as
bench.py runs it), with a camera, and compares in frames/s of the stream
  (a) one multi-dictionary handle with each board bound to its family,
  (b) two single-dictionary handles, each with its own family's boards, over the same frames,
  (c) the multi-dictionary handle of (a) without boards,
in alternating rounds; it reports each configuration's median.

Prints the card name and power limit read in the same run; --out DIR also writes the numbers as JSON.
    python tools/bench_multidict_boards.py [--steps 6] [--runs 3] [--out DIR]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import cv2
import numpy as np
import torch

from bench_marker_refine import card
from bench_multidict import loop
from fiducials_b200 import synth
from fiducials_b200.node import Detector, default_params
import bench_multidict
import multidict_boards_cases as mc

W, H, N, CHUNK = 1920, 1080, 64, 32
A = mc.A
FAMILIES = [A.DICT_5X5_1000, A.DICT_APRILTAG_36h11]


def render(seed):
    rng = np.random.default_rng(seed)
    g = np.full((H, W), 200, np.uint8)
    for k, d in enumerate(FAMILIES):
        x0 = 60 + 940 * k + int(rng.integers(0, 40))
        mc._paste(g, mc._grid_image(d, range(4)), x0, 40 + int(rng.integers(0, 40)))
        mc._paste(g, mc._charuco_image(d, mc.CH_SIZE, mc.CH_PX), x0, 460 + int(rng.integers(0, 40)))
    Hm = np.array([[1 + rng.uniform(-0.03, 0.03), rng.uniform(-0.05, 0.05), rng.uniform(-5, 5)],
                   [rng.uniform(-0.05, 0.05), 1 + rng.uniform(-0.03, 0.03), rng.uniform(-5, 5)],
                   [rng.uniform(-2e-5, 2e-5), rng.uniform(-2e-5, 2e-5), 1.0]])
    g = cv2.warpPerspective(g, Hm, (W, H), flags=cv2.INTER_LINEAR, borderValue=200)
    g = cv2.GaussianBlur(g, (3, 3), 0.7)
    g = np.clip(g + rng.normal(0, 2.0, g.shape), 0, 255).astype(np.uint8)
    return np.ascontiguousarray(cv2.cvtColor(g, cv2.COLOR_GRAY2BGR))


def handles(mode):
    if mode == "b":
        dets = [Detector(default_params(dictionary=d), 0, W, H, CHUNK) for d in FAMILIES]
        for d in dets:
            d.set_boards([mc.grid()])
            d.set_charuco_boards([mc.charuco()])
        return dets
    d = Detector(default_params(dictionary=FAMILIES[0]), 0, W, H, CHUNK)
    d.set_dictionaries([(x, 1000 * k, 0.0) for k, x in enumerate(FAMILIES)])
    if mode == "a":
        d.set_boards([mc.grid(), mc.grid()], [0, 1])
        d.set_charuco_boards([mc.charuco(), mc.charuco()], [0, 1])
    return [d]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: nothing to measure")
    bench_multidict.N, bench_multidict.W, bench_multidict.H = N, W, H
    K, _ = synth.camera_for(W, H)
    frames = [render(700 + i) for i in range(16)]
    dev = torch.from_numpy(np.ascontiguousarray(np.stack([frames[i % 16] for i in range(N)]))).cuda()
    res = {"card": card(), "frames_per_batch": N, "chunk": CHUNK, "dictionaries": FAMILIES, "frames_per_s": {m: [] for m in "abc"}, "markers_per_batch": {}}
    for _ in range(args.runs):  # alternating rounds, each on handles of its own
        for m in "abc":
            dets = handles(m)
            loop(dets, dev, K, 1)  # warm-up
            fps, n_markers = loop(dets, dev, K, args.steps)
            res["frames_per_s"][m].append(round(fps, 1))
            res["markers_per_batch"][m] = n_markers // len(dets)
            if m != "c":
                res.setdefault("board_status", {})[m] = [int(r.status) for d in dets for r in d.last_board_poses()[0]]
            for d in dets:
                d.close()
    res["median_frames_per_s"] = {m: float(np.median(v)) for m, v in res["frames_per_s"].items()}
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_multidict_boards.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
