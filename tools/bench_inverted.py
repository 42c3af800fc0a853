"""Cost of detectInvertedMarker (fid_set_detect_inverted_marker) on bench.py's C2 stream: 128 distinct 1080p frames per batch (two
chunks of 64), frames resident in HBM, DEPTH batches in flight through the same submit/collect loop as bench.py (collect, the records
copied out as a consumer would, the asynchronous map fold; the multi-GPU map merge of bench.py is left out).

Three runs, alternating in one process (ROUNDS x {off, on, on over inverted frames}, each STEPS timed batches after WARMUP batches):
the flag off and on over the normal C2 frames, and on over the same frames inverted (white markers on black).  Medians of the rounds.
Prints the card name and power limit with the numbers; --out DIR also writes them as JSON.
    python tools/bench_inverted.py [--steps 20] [--warmup 3] [--rounds 3] [--out DIR]"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from fiducials_b200 import _lib, synth
from fiducials_b200.node import Detector, FiducialSlam, default_params


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return q.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--depth", type=int, default=2, help="batches in flight (bench.py's FID_BENCH_DEPTH default)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: nothing to measure")

    lib = _lib.load()
    W, H, n_markers, dict_id = synth.CONFIGS["C2"]
    nf, slot = 128, 64
    frames, _, K, D, _ = synth.make_config_stream("C2", nf, seed=0, realizations=8)  # bench.py's stream (rank 0)
    inverted = np.ascontiguousarray(255 - frames)
    det = Detector(default_params(dictionary=dict_id), 0, W, H, slot)
    slam = FiducialSlam(device=0, max_fiducials=512, n_instances=1)
    ident = [0, 0, 0, 0, 0, 0, 1]
    ptrs = {}
    for name, fr in (("normal", frames), ("inverted", inverted)):
        p = C.c_void_p()
        _lib.check(lib.fid_device_alloc(det.h, fr.nbytes, C.byref(p)))
        _lib.check(lib.fid_memcpy_h2d(det.h, p, fr.ctypes.data_as(C.c_void_p), fr.nbytes))
        ptrs[name] = p
    outs = [None] * 4
    state = {"src": "normal"}

    def submit():
        det.submit_batch(ptrs[state["src"]].value, K, D, 0.14, on_device=True, n_frames=nf, width=W, height=H)

    def finish(k):
        outs[k & 3] = det.collect_batch(outs[k & 3])
        counts, _, _, tfs = outs[k & 3]
        slam.update_frames(counts, tfs, ident, ident, asynchronous=True)
        return int(counts.sum())

    def run(steps):
        ahead, total = min(args.depth - 1, steps), 0
        for _ in range(ahead):
            submit()
        for k in range(steps):
            if k + ahead < steps:
                submit()
            total += finish(k)
        slam.sync()
        return total

    MODES = {"off": (False, "normal"), "on": (True, "normal"), "on_inverted": (True, "inverted")}

    def timed(mode):
        on, src = MODES[mode]
        det.set_detect_inverted_marker(on)  # nothing in flight between runs
        state["src"] = src
        run(args.warmup)
        torch.cuda.synchronize()
        _lib.check(lib.fid_timer_start(det.h))
        markers = run(args.steps)
        ms = C.c_float(0)
        _lib.check(lib.fid_timer_stop(det.h, C.byref(ms)))  # device events, as bench.py's device-resident figure
        return nf * args.steps / (ms.value / 1e3), markers / (nf * args.steps)

    fps = {m: [] for m in MODES}
    per_frame = {}
    for m in MODES:  # first-touch warm-up of every path
        timed(m)
    order = list(MODES)
    for r in range(args.rounds):
        for m in (order if r % 2 == 0 else order[::-1]):
            v, mk = timed(m)
            fps[m].append(v)
            per_frame[m] = mk

    res = dict(card=card(), frames_per_batch=nf, steps=args.steps, rounds=args.rounds, markers_per_frame=per_frame, fps=fps,
               median={m: statistics.median(v) for m, v in fps.items()})
    res["on_vs_off_pct"] = 100.0 * (res["median"]["on"] / res["median"]["off"] - 1.0)
    res["on_inverted_vs_off_pct"] = 100.0 * (res["median"]["on_inverted"] / res["median"]["off"] - 1.0)
    print("card: %s" % res["card"])
    for m in MODES:
        print("C2 device-resident frames/s, %-12s %s  median %.0f  (%.1f markers per frame)" % (m + ":", " ".join("%.0f" % v for v in fps[m]), res["median"][m], per_frame[m]))
    print("on vs off %+.2f %%, on over inverted frames vs off %+.2f %%" % (res["on_vs_off_pct"], res["on_inverted_vs_off_pct"]))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_inverted.json"), "w") as fp:
            json.dump(res, fp, indent=1)
    for p in ptrs.values():
        lib.fid_device_free(det.h, p)
    det.close()


if __name__ == "__main__":
    main()
