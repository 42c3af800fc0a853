"""Device time per kernel of bench.py's C2 batch (128 distinct 1080p frames, two chunks of 64, frames resident in HBM), from
torch.profiler with CUDA activities over 4 batches after 3 warm-up batches.  Environment switches of the library (INTEGRATION.md)
apply, e.g. FID_START_PRUNE=1 python tools/kernel_breakdown.py"""
import ctypes as C, os, sys, collections
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from torch.profiler import profile, ProfilerActivity
from fiducials_b200 import _lib, synth
from fiducials_b200.node import Detector, default_params
lib = _lib.load()
W, H, nm, d = synth.CONFIGS["C2"]
nf = 128
frames, truths, K, D, _ = synth.make_config_stream("C2", nf, seed=0, realizations=8)
det = Detector(default_params(dictionary=d), 0, W, H, 64)
dptr = C.c_void_p(); _lib.check(lib.fid_device_alloc(det.h, frames.nbytes, C.byref(dptr))); _lib.check(lib.fid_memcpy_h2d(det.h, dptr, frames.ctypes.data_as(C.c_void_p), frames.nbytes))
run = lambda: det.detect_pose_batch(dptr.value, K, D, 0.14, on_device=True, n_frames=nf, width=W, height=H)
for _ in range(3):
    run()
torch.cuda.synchronize()
NB = 4
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(NB):
        run()
    torch.cuda.synchronize()
tot = collections.Counter(); cnt = collections.Counter()
for e in prof.events():
    t = getattr(e, "device_time_total", None)
    if t is None:
        t = getattr(e, "cuda_time_total", 0)
    name = e.name.split("(")[0].replace("void ", "")
    tot[name] += t; cnt[name] += 1
all_us = sum(tot.values())
print(torch.cuda.get_device_name(0), "-- per batch of %d frames (2 chunks of 64), kernel device time summed over launches" % nf)
for k, v in tot.most_common(25):
    print("%-60s %9.3f ms/batch %5.1f %%  launches/batch %.1f" % (k[:60], v / 1e3 / NB, 100 * v / all_us, cnt[k] / NB))
print("sum %.3f ms/batch" % (all_us / 1e3 / NB))
print("stage_ms", {k: round(v, 3) for k, v in det.last_stage_ms().items() if v > 0.001})
print("counters", det.last_counters())
lib.fid_device_free(det.h, dptr)
det.close()
