"""Cost of the opt-in marker confidence (fid_set_marker_confidence) on bench.py's C2 stream: 128 distinct 1080p frames per batch
(two chunks of 64), frames resident in HBM, DEPTH batches in flight through the same submit/collect loop as bench.py (collect, the
records copied out as a consumer would, the asynchronous map fold; the multi-GPU map merge of bench.py is left out).

1. device-resident frames/s with the option off and on, alternating in one process (ROUNDS x {off, on}, each STEPS timed batches
   after WARMUP batches), so both modes see the same card state;
2. in separate runs under torch.profiler, off and on: device time per 128-frame batch of the identification kernels
   (k_identify_first, k_identify_retry; their confidence variants when on) and of k_conf_gather.

Prints the card name and power limit with the numbers; --out DIR also writes them as JSON.
    python tools/bench_confidence.py [--steps 20] [--warmup 3] [--rounds 4] [--out DIR]"""
import argparse
import collections
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch.profiler import ProfilerActivity, profile

from fiducials_b200 import _lib, synth
from fiducials_b200.node import MAXM, Detector, FiducialSlam, default_params


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
    confs = (C.c_float * (nf * MAXM))()
    n_frames = C.c_int(0)
    outs = [None] * 4
    state = {"on": False, "markers": 0}

    def submit():
        det.submit_batch(dptr.value, K, D, 0.14, on_device=True, n_frames=nf, width=W, height=H)

    def finish(k):
        outs[k & 3] = det.collect_batch(outs[k & 3])
        counts, _, _, tfs = outs[k & 3]
        if state["on"]:
            _lib.check(lib.fid_last_marker_confidence(det.h, MAXM, C.byref(n_frames), C.cast(confs, C.c_void_p)))
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

    def timed(on):
        state["on"] = on
        det.set_marker_confidence(on)  # nothing in flight between runs
        run(args.warmup)
        torch.cuda.synchronize()
        _lib.check(lib.fid_timer_start(det.h))
        markers = run(args.steps)
        ms = C.c_float(0)
        _lib.check(lib.fid_timer_stop(det.h, C.byref(ms)))  # device events, as bench.py's device-resident figure
        state["markers"] = markers
        return nf * args.steps / (ms.value / 1e3)

    fps = {False: [], True: []}
    timed(False)  # first-touch warm-up of both paths
    timed(True)
    for r in range(args.rounds):
        for on in ((False, True) if r % 2 == 0 else (True, False)):
            fps[on].append(timed(on))

    # kernel device times, a profiler run of its own per mode
    NB = 4
    KERNELS = ("k_identify_first", "k_identify_retry", "k_conf_gather", "k_finish")
    kern = {}
    for on in (False, True):
        state["on"] = on
        det.set_marker_confidence(on)
        run(args.warmup)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run(NB)
            torch.cuda.synchronize()
        tot, cnt = collections.Counter(), collections.Counter()
        for e in prof.events():
            t = getattr(e, "device_time_total", None)
            if t is None:
                t = getattr(e, "cuda_time_total", 0)
            name = e.name.split("(")[0].replace("void ", "").replace("fid::", "").split("<")[0]
            tot[name] += t
            cnt[name] += 1
        kern["on" if on else "off"] = {k: dict(ms_per_batch=tot[k] / 1e3 / NB, launches_per_batch=cnt[k] / NB) for k in KERNELS}
        kern["on" if on else "off"]["all_kernels_ms_per_batch"] = sum(v for k, v in tot.items() if k.startswith("k_")) / 1e3 / NB

    res = dict(card=card(), frames_per_batch=nf, steps=args.steps, rounds=args.rounds, markers_per_frame=state["markers"] / (nf * args.steps),
               fps_off=fps[False], fps_on=fps[True], median_off=statistics.median(fps[False]), median_on=statistics.median(fps[True]),
               kernels=kern)
    res["on_vs_off_pct"] = 100.0 * (res["median_on"] / res["median_off"] - 1.0)
    print("card: %s" % res["card"])
    print("C2 device-resident frames/s, option off: %s  median %.0f" % (" ".join("%.0f" % v for v in fps[False]), res["median_off"]))
    print("C2 device-resident frames/s, option on:  %s  median %.0f  (%+.2f %%)" % (" ".join("%.0f" % v for v in fps[True]), res["median_on"], res["on_vs_off_pct"]))
    for mode in ("off", "on"):
        for k in KERNELS:
            v = kern[mode][k]
            print("%-3s %-18s %.4f ms per %d-frame batch (%.1f launches)" % (mode, k, v["ms_per_batch"], nf, v["launches_per_batch"]))
        print("%-3s all kernels %.3f ms per batch" % (mode, kern[mode]["all_kernels_ms_per_batch"]))
    print("%.1f markers per frame" % res["markers_per_frame"])
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_confidence.json"), "w") as fp:
            json.dump(res, fp, indent=1)
    lib.fid_device_free(det.h, dptr)
    det.close()


if __name__ == "__main__":
    main()
