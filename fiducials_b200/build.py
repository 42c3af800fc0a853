"""In-tree build of libfiducials_b200.so (nvcc, sm_90a only).  Used by __graft_entry__.build()."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libfiducials_b200.so")
SOURCES = ["fid_api.cu", "fid_map.cu", "fid_map_refine.cu", "fid_map_ba.cu", "fid_map_localize.cu", "fid_jpeg.cu", "fid_calib.cu"]
# --fmad=false: OpenCV's float32/float64 arithmetic (cornerSubPix, perimeters, the LM trajectory) is
# compiled without FMA contraction on x86-64; contracting here would change iteration counts.
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "--fmad=false", "-std=c++17", "-Xcompiler", "-fPIC", "-shared"]


def _newest_source():
    t = 0.0
    for root in (CSRC, os.path.join(os.path.dirname(HERE), "include")):
        for f in os.listdir(root):
            if f.endswith((".cu", ".cuh", ".h", ".hpp")):
                t = max(t, os.path.getmtime(os.path.join(root, f)))
    return t


def build(force=False, verbose=False):
    if not force and os.path.exists(OUT) and os.path.getmtime(OUT) >= _newest_source():
        return OUT
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", OUT] + [os.path.join(CSRC, s) for s in SOURCES]
    print("[fiducials_b200] " + " ".join(cmd), file=sys.stderr)
    subprocess.check_call(cmd)
    return OUT


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose="-v" in sys.argv)
