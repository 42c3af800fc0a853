"""Cost of the opt-in ChArUco stage (fid_set_charuco_boards) on one GPU.

1. C2 device-resident frames/s with no ChArUco board and with one, alternating in one process (ROUNDS x {off, on}, each STEPS
   timed batches after WARMUP batches), through the same submit/collect loop as bench.py: 128 distinct 1080p frames per batch (two
   chunks of 64) of bench.py's C2 stream, DEPTH batches in flight, the asynchronous map fold (the multi-GPU merge is left out).
   The board is a 25 x 20 ChArUco board holding all 250 ids of DICT_6X6_250, so every detected marker is one of its markers and
   its nearest corners are interpolated and refined (the stream's markers are not laid out as that board: the worst case for the
   corner count, not a meaningful detection).
2. In a separate run under torch.profiler: device time of k_charuco (and k_finish, for scale) per 128-frame batch of rendered 1080p
   ChArUco frames (a 7 x 5 board, cv2.aruco.CharucoBoard.generateImage warped into each frame at a seeded pose), with a camera.

Prints the card name and power limit read in the same run; --out DIR also writes the numbers as JSON.
    python tools/bench_charuco.py [--steps 20] [--warmup 3] [--rounds 4] [--out DIR]"""
import argparse
import collections
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cv2
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

from fiducials_b200 import _lib, synth
from fiducials_b200.board import charuco_board
from fiducials_b200.node import Detector, FiducialSlam, default_params


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return q.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def rendered_charuco_frames(n, W, H, K, board, seed=0):
    """n BGR frames, each with the ChArUco board warped in at a seeded pose facing the camera (tilted up to ~20 degrees)."""
    rng = np.random.default_rng(seed)
    cvb = cv2.aruco.CharucoBoard(board.size, board.square_length, board.marker_length, cv2.aruco.getPredefinedDictionary(cv2.aruco.DICT_6X6_250),
                                 np.asarray(board.ids, np.int32))
    px = 80
    img = cvb.generateImage((board.size[0] * px + px, board.size[1] * px + px), marginSize=px // 2, borderBits=1)
    s = board.square_length / px
    A = np.array([[s, 0, -px // 2 * s], [0, s, -px // 2 * s], [0, 0, 1]])
    c = np.array([board.size[0] * board.square_length / 2, board.size[1] * board.square_length / 2, 0.0])
    out = np.empty((n, H, W, 3), np.uint8)
    for f in range(n):
        R = cv2.Rodrigues(rng.normal(0, 0.2, 3) * np.array([1, 1, 0.5]))[0]
        z = rng.uniform(0.5, 0.9)
        u, v = rng.uniform(0.35 * W, 0.65 * W), rng.uniform(0.35 * H, 0.65 * H)
        t = z * np.array([(u - K[0, 2]) / K[0, 0], (v - K[1, 2]) / K[1, 1], 1.0]) - R @ c
        Hm = K @ np.column_stack([R[:, 0], R[:, 1], t]) @ A
        g = cv2.warpPerspective(img, Hm, (W, H), flags=cv2.INTER_LINEAR, borderValue=128)
        out[f] = cv2.cvtColor(cv2.GaussianBlur(g, (5, 5), 1.0), cv2.COLOR_GRAY2BGR)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--depth", type=int, default=2, help="batches in flight (bench.py's FID_BENCH_DEPTH default)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: nothing to measure")

    lib = _lib.load()
    W, H, n_markers, dict_id = synth.CONFIGS["C2"]
    nf, slot = 128, 64
    frames, _, K, D, _ = synth.make_config_stream("C2", nf, seed=0, realizations=8)  # bench.py's stream (rank 0)
    det = Detector(default_params(dictionary=dict_id), 0, W, H, slot)
    slam = FiducialSlam(device=0, max_fiducials=512, n_instances=1)
    ident = [0, 0, 0, 0, 0, 0, 1]
    dptr = C.c_void_p()
    _lib.check(lib.fid_device_alloc(det.h, frames.nbytes, C.byref(dptr)))
    _lib.check(lib.fid_memcpy_h2d(det.h, dptr, frames.ctypes.data_as(C.c_void_p), frames.nbytes))
    big = charuco_board((25, 20), 0.04, 0.03)  # ids 0..249: every marker of DICT_6X6_250
    outs = [None] * 4
    state = {"on": False, "markers": 0, "corners": 0}

    def submit(ptr):
        det.submit_batch(ptr, K, D, 0.14, on_device=True, n_frames=nf, width=W, height=H)

    def finish(k):
        outs[k & 3] = det.collect_batch(outs[k & 3])
        counts, _, _, tfs = outs[k & 3]
        if state["on"]:
            state["corners"] += sum(int(r.n_corners) for fr in det.last_charuco() for r, _, _ in fr)
        slam.update_frames(counts, tfs, ident, ident, asynchronous=True)
        return int(counts.sum())

    def run(steps, ptr):
        ahead, total = min(args.depth - 1, steps), 0
        for _ in range(ahead):
            submit(ptr)
        for k in range(steps):
            if k + ahead < steps:
                submit(ptr)
            total += finish(k)
        slam.sync()
        return total

    def timed(on):
        state["on"] = on
        det.set_charuco_boards([big] if on else [])  # nothing in flight between runs
        run(args.warmup, dptr.value)
        torch.cuda.synchronize()
        _lib.check(lib.fid_timer_start(det.h))
        markers = run(args.steps, dptr.value)
        ms = C.c_float(0)
        _lib.check(lib.fid_timer_stop(det.h, C.byref(ms)))  # device events, as bench.py's device-resident figure
        state["markers"] = markers
        return nf * args.steps / (ms.value / 1e3)

    fps = {False: [], True: []}
    timed(False)  # first-touch warm-up of both paths
    timed(True)
    state["corners"] = 0
    for r in range(args.rounds):
        for on in ((False, True) if r % 2 == 0 else (True, False)):
            fps[on].append(timed(on))
    c2_corners = state["corners"] / (nf * args.steps * args.rounds)

    # k_charuco device time on rendered ChArUco frames, profiler run of its own
    small = charuco_board((7, 5), 0.04, 0.03)
    ch_frames = np.ascontiguousarray(rendered_charuco_frames(nf, W, H, K, small))
    cptr = C.c_void_p()
    _lib.check(lib.fid_device_alloc(det.h, ch_frames.nbytes, C.byref(cptr)))
    _lib.check(lib.fid_memcpy_h2d(det.h, cptr, ch_frames.ctypes.data_as(C.c_void_p), ch_frames.nbytes))
    state["on"] = True
    det.set_charuco_boards([small])
    run(args.warmup, cptr.value)
    state["corners"] = 0
    torch.cuda.synchronize()
    NB = 4
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(NB, cptr.value)
        torch.cuda.synchronize()
    tot, cnt = collections.Counter(), collections.Counter()
    for e in prof.events():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = getattr(e, "cuda_time_total", 0)
        name = e.name.split("(")[0].replace("void ", "").replace("fid::", "")
        tot[name] += t
        cnt[name] += 1
    kern = {k: dict(ms_per_batch=tot[k] / 1e3 / NB, launches_per_batch=cnt[k] / NB) for k in ("k_charuco", "k_finish")}
    rendered_corners = state["corners"] / (nf * NB)

    res = dict(card=card(), frames_per_batch=nf, steps=args.steps, rounds=args.rounds, markers_per_frame=state["markers"] / (nf * args.steps),
               fps_off=fps[False], fps_on=fps[True], median_off=statistics.median(fps[False]), median_on=statistics.median(fps[True]),
               c2_charuco_corners_per_frame=c2_corners, rendered_charuco_corners_per_frame=rendered_corners, kernels=kern)
    res["on_vs_off_pct"] = 100.0 * (res["median_on"] / res["median_off"] - 1.0)
    print("card: %s" % res["card"])
    print("C2 device-resident frames/s, no ChArUco board: %s  median %.0f" % (" ".join("%.0f" % v for v in fps[False]), res["median_off"]))
    print("C2 device-resident frames/s, 25x20 board:      %s  median %.0f  (%+.2f %%), %.1f corners per frame"
          % (" ".join("%.0f" % v for v in fps[True]), res["median_on"], res["on_vs_off_pct"], c2_corners))
    for k, v in kern.items():
        print("%-12s %.4f ms per %d-frame batch of rendered 7x5 ChArUco frames (%.1f launches; %.1f corners per frame)"
              % (k, v["ms_per_batch"], nf, v["launches_per_batch"], rendered_corners))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_charuco.json"), "w") as fp:
            json.dump(res, fp, indent=1)
    lib.fid_device_free(det.h, cptr)
    lib.fid_device_free(det.h, dptr)
    det.close()


if __name__ == "__main__":
    main()
