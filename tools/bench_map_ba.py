"""fid_map_bundle_adjust's cost on the device: synth.make_c5_sequence's 500-marker ceiling (25 x 20 at 1 m pitch) at 1 000 and 10 000
frames, 10 markers per frame, corners projected with 0.5 px noise and the start map perturbed as the fold leaves it.  Reports the
device ms of the call, the iterations and ms per LM step split by kernel family from a torch.profiler run of its own (eval:
k_ba_eval / k_ba_sums / k_ba_lm; Schur build: k_ba_factor / k_ba_z / k_ba_clear / k_ba_reduce / k_ba_rhs; Cholesky: k_dense_*;
back-substitution: k_ba_backsub; trial: k_ba_trial / k_ba_decide), fid_map_refine's time on the equivalent messages (the same
frames' per-marker poses from fid_pose), whether the run ended on the relative-step test (converged) or at max_iter, and the card's
name and power limit from the same run.  --scipy times scipy.optimize.least_squares (the CPU arm) against the call on a 30-marker,
150-frame scene: its dense trust-region solve does not fit C5's ~9 000 parameters.  Writes one JSON line per workload to stdout and, with --out, to a file."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))

import map_ba_cases as mc  # noqa: E402
from fiducials_b200 import _lib  # noqa: E402
from fiducials_b200.node import Detector, FiducialSlam  # noqa: E402

FAMILIES = {"eval": ("k_ba_eval", "k_ba_sums", "k_ba_lm"), "schur": ("k_ba_factor", "k_ba_z", "k_ba_clear", "k_ba_reduce", "k_ba_rhs"),
            "cholesky": ("k_dense_potrf", "k_dense_trsm", "k_dense_syrk"), "backsub": ("k_ba_backsub",), "trial": ("k_ba_trial", "k_ba_decide"),
            "solve_trsv": ("k_dense_trsv",), "init": ("k_ba_init",), "final_std": ("k_ba_eye", "k_ba_std")}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        return q.splitlines()[0] if q else "unknown"
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def run(sc, slam_cap=512):
    s = FiducialSlam(max_fiducials=slam_cap)
    s.loadMap(mc.file_entries(sc))
    t0 = time.perf_counter()
    st, rv, tv, status, sd = s.bundle_adjust(sc["counts"], sc["fids"], sc["corners"], sc["K"], sc["D"], sc["fiducial_len"])
    return st, time.perf_counter() - t0


def refine_time(sc):
    det = Detector(max_width=64, max_height=64)
    msgs = []
    for f in range(len(sc["counts"])):
        n = int(sc["counts"][f])
        out = det.pose(sc["fids"][f, :n], sc["corners"][f, :n], sc["K"], sc["D"], sc["fiducial_len"])
        msgs.append([dict(fiducial_id=int(t.fiducial_id), translation=list(t.translation), rotation=list(t.rotation), image_error=t.image_error,
                          object_error=t.object_error, fiducial_area=t.fiducial_area) for t in out])
    s = FiducialSlam(max_fiducials=512)
    s.loadMap(mc.file_entries(sc))
    s.refine(msgs)  # warm-up
    s = FiducialSlam(max_fiducials=512)
    s.loadMap(mc.file_entries(sc))
    st = s.refine(msgs)
    return st.solve_ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, nargs="+", default=[1000, 10000])
    ap.add_argument("--profile", action="store_true", help="split the device time by kernel family with torch.profiler (a run of its own)")
    ap.add_argument("--scipy", action="store_true", help="the CPU arm: scipy on a 30-marker x 150-frame scene against the call")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = card()
    lines = []
    for nf in a.frames:
        sc = mc.make_scene(0, n_markers=500, n_frames=nf, visible=10, noise=0.5, size=(1920, 1080), f=500.0)
        run(mc.make_scene(1, n_markers=16, n_frames=40))  # warm-up: module load, first launches
        st, wall = run(sc)
        r = dict(workload=f"c5_500m_{nf}f", card=gpu, device_ms=st.device_ms, wall_s=wall, iterations=st.iterations, steps=st.n_steps,
                 ms_per_step=st.device_ms / max(st.n_steps, 1), frames=st.frames_used, markers=st.markers_used, observations=st.observations_used,
                 initial_rms=st.initial_rms, final_rms=st.final_rms, kernel_launches=st.kernel_launches, converged=st.converged, refine_ms=refine_time(sc))
        if a.profile:
            import torch
            from torch.profiler import ProfilerActivity, profile

            torch.cuda.init()
            with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
                st2, _ = run(sc)
            tot = {k: 0.0 for k in FAMILIES}
            for ev in prof.key_averages():
                for k, names in FAMILIES.items():
                    if any(n in ev.key for n in names):
                        tot[k] += ev.device_time_total / 1000.0 if hasattr(ev, "device_time_total") else ev.cuda_time_total / 1000.0
            r["profile_ms"] = tot
            r["profile_ms_per_step"] = {k: v / max(st2.n_steps, 1) for k, v in tot.items()}
        print(json.dumps(r), flush=True)
        lines.append(r)
    if a.scipy:
        sc = mc.make_scene(7, n_markers=30, n_frames=150, dist=True, oblique=True)
        st, _ = run(sc)
        h = mc.hs_bundle_adjust(sc, criteria="init")
        used = [f for f in range(150) if h["status"][f] == 1]
        t0 = time.perf_counter()
        ref = mc.scipy_bundle_adjust(sc, {f: mc.rot(h["rvecs"][f]) for f in used}, {f: h["tvecs"][f] for f in used})
        r = dict(workload="scipy_30m_150f", card=gpu, device_ms=st.device_ms, iterations=st.iterations, converged=st.converged, scipy_s=time.perf_counter() - t0,
                 scipy_nfev=ref["nfev"], cost_rel_diff=abs(st.final_rms ** 2 * 4 * st.observations_used / ref["cost"] - 1))
        print(json.dumps(r), flush=True)
        lines.append(r)
    if a.out:
        with open(a.out, "w") as fh:
            for r in lines:
                fh.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
