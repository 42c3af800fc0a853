"""Cost of the start-queue replay (kernels_contour.cuh, k_rescan_starts): fid_detect on the half-checkerboard 1920 x 1080 frame of
tests/contour_cases.py, whose start cracks overflow the queue of a one-frame handle (max_batch 1, replayed) but fit the pooled queue of
a four-frame handle (max_batch 4, walked once), and on the C2 frame that overflows neither.  Host clock around the synchronous call,
median of --reps calls after --warmup.  Also fid_create's device memory (torch.cuda.mem_get_info before and after) for the C2 bench
handle.  The C2 frame's time with max_batch 1 is the latency a one-frame caller pays for the replay launches that return at once.
Prints one JSON line with the GPU's name and power limit.

    python tools/replay_cost.py [--reps 50] [--warmup 5]
"""
import argparse, json, os, statistics, subprocess, sys, time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch

    import contour_cases as cc
    from fiducials_b200 import _lib, synth
    from fiducials_b200.node import Detector, default_params

    torch.cuda.init()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    torch.cuda.synchronize()
    free0, _ = torch.cuda.mem_get_info()
    det = Detector(default_params(dictionary=10), 0, 1920, 1080, 64)  # bench.py's C2 handle
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    det.close()
    out = {"gpu": gpu, "fid_create_bytes_c2_batch64": free0 - free1}
    frames = {"checker1_half_fhd": cc.render("checker1_half_fhd")[0], "c2": synth.make_config_frame("C2", 3)[0]}
    for max_batch in (1, 4):
        det = Detector(default_params(dictionary=cc.DICT), 0, 1920, 1080, max_batch)
        for name, bgr in frames.items():
            try:
                for _ in range(args.warmup):
                    det.detect(bgr)
            except _lib.FidError as e:  # a library without the replay: the overflowing frame fails
                out[f"{name}_max_batch{max_batch}_ms"] = str(e)
                continue
            t = []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                det.detect(bgr)
                t.append((time.perf_counter() - t0) * 1e3)
            out[f"{name}_max_batch{max_batch}_ms"] = round(statistics.median(t), 3)
        det.close()
    if isinstance(out["checker1_half_fhd_max_batch1_ms"], float):
        out["replay_ms"] = round(out["checker1_half_fhd_max_batch1_ms"] - out["checker1_half_fhd_max_batch4_ms"], 3)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
