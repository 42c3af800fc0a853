"""Cost of the recovery of missed board markers inside the batch calls (fid_set_batch_marker_refinement) on one GPU.

Two workloads, each a 128-frame batch of 1080p frames in device memory, run in chunks of 64 through the submit/collect loop with two
batches in flight (as bench.py runs it), with a camera:
  * boards: the rendered frames of tools/bench_marker_refine.py (a 10 x 7 GridBoard, three markers' inner bits painted over);
  * c2: bench.py's C2 stream (16 markers per frame from a 250-id dictionary) with one 25 x 10 board of all 250 ids set, the worst
    case for the board stages: every marker is on the board and the stream's markers are not laid out as the board.
Per workload: the device time of k_rejected, k_marker_refine and k_recovered_pose per 128-frame batch (torch.profiler, a run of
its own), then frames/s with refinement off and on on the same handle, in alternating runs.

Prints the card name and power limit read in the same run; --out DIR also writes the numbers as JSON.
    python tools/bench_batch_refine.py [--steps 10] [--runs 3] [--out DIR]"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

from bench_marker_refine import DICT, LENGTH, SEP, SIZE, card, rendered_frames
from fiducials_b200 import synth
from fiducials_b200.board import grid_board
from fiducials_b200.node import Detector, default_params

W, H, N, CHUNK = 1920, 1080, 128, 64
KERNELS = ("k_rejected", "k_marker_refine", "k_recovered_pose")


def frames_boards():
    K, _ = synth.camera_for(W, H)
    board = grid_board(SIZE, LENGTH, SEP)
    g = rendered_frames(N, W, H, K, board)
    return np.ascontiguousarray(np.repeat(np.stack(g)[..., None], 3, axis=3)), K, board, DICT


def frames_c2():
    fr = [synth.make_config_frame("C2", s) for s in range(16)]
    K, d = fr[0][2], fr[0][4]
    frames = np.ascontiguousarray(np.stack([fr[i % 16][0] for i in range(N)]))
    return frames, K, grid_board((25, 10), 0.05, 0.01, list(range(250))), d


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


def measure(name, make, steps, runs):
    frames, K, board, d = make()
    dev = torch.from_numpy(frames).cuda()
    det = Detector(default_params(dictionary=d), 0, W, H, CHUNK)
    det.set_boards([board])
    det.set_marker_refinement()
    det.set_batch_marker_refinement(True)
    loop(det, dev, K, 2)  # warm-up
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        loop(det, dev, K, 1)  # two batches
        torch.cuda.synchronize()
    dev_ms = {k: sum(e.device_time for e in prof.events() if k + "(" in e.name) / 1000.0 / 2 for k in KERNELS + ("k_finish",)}
    recovered = sum(len(r[0]) for r in det.last_marker_refinement())
    fps = {"off": [], "on": []}
    for _ in range(runs):
        for mode in ("off", "on"):
            det.set_batch_marker_refinement(mode == "on")
            loop(det, dev, K, 1)
            fps[mode].append(round(loop(det, dev, K, steps)[0], 1))
    det.close()
    return {"workload": name, "device_ms_per_batch": dev_ms, "recovered_per_batch": recovered, "frames_per_s": fps,
            "median_off": float(np.median(fps["off"])), "median_on": float(np.median(fps["on"]))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: nothing to measure")
    res = {"card": card(), "frames_per_batch": N, "chunk": CHUNK}
    res["results"] = [measure("boards", frames_boards, args.steps, args.runs), measure("c2", frames_c2, args.steps, args.runs)]
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_batch_refine.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
