"""Cost of the recovery of missed board markers (fid_set_marker_refinement, fid_refine_detected_markers) on one GPU.

128 rendered 1080p frames, each with a 10 x 7 GridBoard of DICT_6X6_250 (40 mm markers, 10 mm gaps) warped in at a seeded pose and
three of its markers' inner bits painted over; cv2's detectMarkers gives each frame's detected and rejected lists.  Under
torch.profiler, one fid_refine_detected_markers call per frame (with a camera), after a warm-up pass: the device time of
k_marker_refine summed over the 128 frames, and the markers recovered.  The batch path and its frames/s are measured by
tools/bench_batch_refine.py.

Prints the card name and power limit read in the same run; --out DIR also writes the numbers as JSON.
    python tools/bench_marker_refine.py [--frames 128] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cv2
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

from fiducials_b200 import synth
from fiducials_b200.board import grid_board
from fiducials_b200.node import Detector, default_params
from oracle import aruco_oracle as ao

DICT = cv2.aruco.DICT_6X6_250
SIZE, LENGTH, SEP = (10, 7), 0.04, 0.01


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return q.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def rendered_frames(n, W, H, K, board, seed=0):
    """n gray frames with the board at a seeded pose facing the camera and three markers' inner bits painted over."""
    rng = np.random.default_rng(seed)
    d = cv2.aruco.getPredefinedDictionary(DICT)
    px = 60
    mpp = LENGTH / px
    margin = px // 2
    w = int(round((SIZE[0] * LENGTH + (SIZE[0] - 1) * SEP) / mpp)) + 2 * margin
    h = int(round((SIZE[1] * LENGTH + (SIZE[1] - 1) * SEP) / mpp)) + 2 * margin
    img = cv2.aruco.GridBoard(SIZE, LENGTH, SEP, d).generateImage((w, h), marginSize=margin, borderBits=1)
    A = np.array([[mpp, 0, -margin * mpp], [0, mpp, -margin * mpp], [0, 0, 1]])
    c = np.array([(SIZE[0] * (LENGTH + SEP) - SEP) / 2, (SIZE[1] * (LENGTH + SEP) - SEP) / 2, 0.0])
    ms = d.markerSize
    out = []
    for _ in range(n):
        R = cv2.Rodrigues(rng.normal(0, 0.2, 3) * np.array([1, 1, 0.5]))[0]
        z = rng.uniform(0.6, 1.0)
        u, v = rng.uniform(0.4 * W, 0.6 * W), rng.uniform(0.4 * H, 0.6 * H)
        t = z * np.array([(u - K[0, 2]) / K[0, 0], (v - K[1, 2]) / K[1, 1], 1.0]) - R @ c
        P = K @ np.column_stack([R[:, 0], R[:, 1], t])
        g = cv2.warpPerspective(img, P @ A, (W, H), flags=cv2.INTER_LINEAR, borderValue=128)
        for k in rng.choice(len(board.ids), 3, replace=False):  # a band of two code rows painted over
            o = board.obj_points[k].astype(np.float64)
            du, dv = (o[1] - o[0]) / (ms + 2), (o[3] - o[0]) / (ms + 2)
            r0 = int(rng.integers(1, ms - 1))
            quad = [o[0] + du + dv * r0, o[0] + du * (ms + 1) + dv * r0, o[0] + du * (ms + 1) + dv * (r0 + 2), o[0] + du + dv * (r0 + 2)]
            p = np.array([P @ np.array([q[0], q[1], 1.0]) for q in quad])
            cv2.fillConvexPoly(g, np.round(p[:, :2] / p[:, 2:] * 16).astype(np.int32), 255, lineType=cv2.LINE_AA, shift=4)
        out.append(cv2.GaussianBlur(g, (3, 3), 0.8))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=128)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: nothing to measure")
    W, H = 1920, 1080
    K, _ = synth.camera_for(W, H)
    D = np.zeros(5)
    board = grid_board(SIZE, LENGTH, SEP)
    frames = rendered_frames(args.frames, W, H, K, board)
    cvdet = cv2.aruco.ArucoDetector(cv2.aruco.getPredefinedDictionary(DICT), ao.reference_detector_params())
    inputs = []
    for g in frames:
        corners, ids, rej = cvdet.detectMarkers(g)
        ids = np.zeros(0, np.int32) if ids is None else ids.reshape(-1).astype(np.int32)
        inputs.append((cv2.cvtColor(g, cv2.COLOR_GRAY2BGR), ids, np.array(corners, np.float32).reshape(-1, 4, 2), np.array(rej, np.float32).reshape(-1, 4, 2)))
    det = Detector(default_params(dictionary=DICT), 0, W, H, 1)
    det.set_boards([board])
    det.set_marker_refinement()

    def run():
        rec = 0
        for bgr, ids, corners, rej in inputs:
            rec += len(det.refine_markers(bgr, ids, corners, rej, K, D)[3])
        return rec

    run()  # warm-up
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        recovered = run()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.name.endswith("k_marker_refine(fid::MarkerRefineArgs)") or "k_marker_refine" in e.name]
    total_ms = sum(e.device_time for e in ev) / 1000.0
    res = {
        "card": card(),
        "frames": len(inputs),
        "launches": len(ev),
        "detected_markers": int(sum(len(i[1]) for i in inputs)),
        "rejected_candidates": int(sum(len(i[3]) for i in inputs)),
        "recovered_markers": recovered,
        "k_marker_refine_ms_total": total_ms,
        "k_marker_refine_us_per_frame": 1000.0 * total_ms / max(len(ev), 1),
    }
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_marker_refine.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
