"""A/B of built libraries on the border walk: for every NAME=path/to/libfiducials_b200.so given, alternating between them
`--reps` times in one process tree, run tools/kernel_breakdown.py (device time of k_walk, k_emit and k_threshold per 128-frame C2
batch) and `bench.py --gpus 1 --steps 20 --warmup 3` (C2 frames/s, CPU baseline skipped), the last run of each library with
--dump-outputs; print per library the runs, their median and range, and whether the dumps are byte-identical with the first
library's.  The library under test is copied over the package's own, which is put back at the end.

    python tools/ab_walk.py parent=ab_libs/parent.so new=fiducials_b200/libfiducials_b200.so
    python tools/ab_walk.py --reps 1 --no-bench a=... b=... c=...          # kernel times only
    python tools/ab_walk.py --reps 1 --no-breakdown --workload C4 a=... b=...
"""
import argparse, filecmp, json, os, re, shutil, statistics, subprocess, sys, tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "fiducials_b200", "libfiducials_b200.so")
KERNELS = ("k_walk", "k_emit", "k_threshold")


def run(cmd, env=None):
    p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    if p.returncode != 0:
        raise SystemExit("%s failed (%d):\n%s\n%s" % (" ".join(cmd), p.returncode, p.stdout[-2000:], p.stderr[-4000:]))
    return p.stdout


def breakdown():
    out = run([sys.executable, os.path.join("tools", "kernel_breakdown.py")])
    ms = dict.fromkeys(KERNELS, 0.0)
    for line in out.splitlines():
        m = re.match(r"(.+?)\s+([0-9.]+) ms/batch", line)
        if m:
            for k in KERNELS:
                if re.search(r"\b%s\b" % k, m.group(1).replace("fid::", "").split("<")[0]):
                    ms[k] += float(m.group(2))
    return ms


def bench(workload, dump):
    env = dict(os.environ, FID_BENCH_SKIP_CPU="1")
    cmd = [sys.executable, "bench.py", "--gpus", "1", "--steps", "20", "--warmup", "3", "--workload", workload]
    if dump:
        cmd += ["--dump-outputs", dump]
    d = json.loads(run(cmd, env).strip().splitlines()[-1])
    stage = d.get("roofline", {}).get("stage_ms_per_batch", {})
    return {"value": d["value"], "e2e": d["e2e"]["value"], "walk_r3": stage.get("walk_r3"), "parity": d.get("parity", {}).get("parity_checked_frames")}


def same_tree(a, b):
    c = filecmp.dircmp(a, b)
    if c.left_only or c.right_only or c.funny_files:
        return False
    _, mismatch, errors = filecmp.cmpfiles(a, b, c.common_files, shallow=False)
    return not mismatch and not errors and all(same_tree(os.path.join(a, s), os.path.join(b, s)) for s in c.common_dirs)


def summary(xs):
    xs = [x for x in xs if x is not None]
    if not xs:
        return "-"
    return "median %.3f  range %.3f .. %.3f  runs %s" % (statistics.median(xs), min(xs), max(xs), " ".join("%.3f" % x for x in xs))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs="+", metavar="NAME=PATH")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--workload", default="C2")
    ap.add_argument("--no-bench", action="store_true")
    ap.add_argument("--no-breakdown", action="store_true")
    args = ap.parse_args()
    libs = [(s.split("=", 1)[0], os.path.abspath(s.split("=", 1)[1])) for s in args.libs]
    print(run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"]).strip())
    tmp = tempfile.mkdtemp(prefix="ab_walk_")
    keep = os.path.join(tmp, "own.so")
    if os.path.exists(LIB):
        shutil.copy2(LIB, keep)
    staged = {}
    for name, path in libs:  # the package's own library may be one of the candidates: take copies before overwriting it
        staged[name] = os.path.join(tmp, name + ".so")
        shutil.copy2(path, staged[name])
    kern = {n: {k: [] for k in KERNELS} for n, _ in libs}
    runs = {n: [] for n, _ in libs}
    try:
        for rep in range(args.reps):
            for name, _ in libs:
                shutil.copy2(staged[name], LIB)
                if not args.no_breakdown:
                    ms = breakdown()
                    for k in KERNELS:
                        kern[name][k].append(ms[k])
                if not args.no_bench:
                    last = rep == args.reps - 1
                    runs[name].append(bench(args.workload, os.path.join(tmp, "dump_" + name) if last else None))
                print("rep %d %s: %s %s" % (rep, name, {k: v[-1] for k, v in kern[name].items() if v}, runs[name][-1] if runs[name] else ""), flush=True)
    finally:
        if os.path.exists(keep):
            shutil.copy2(keep, LIB)
    print("\n== %s, %d alternating runs each ==" % (args.workload, args.reps))
    for name, _ in libs:
        print(name)
        if not args.no_breakdown:
            for k in KERNELS:
                print("  %-12s ms per 128-frame batch: %s" % (k, summary(kern[name][k])))
        if not args.no_bench:
            print("  frames/s (device-resident): %s" % summary([r["value"] for r in runs[name]]))
            print("  frames/s (end to end):      %s" % summary([r["e2e"] for r in runs[name]]))
            print("  walk_r3 stage ms per batch: %s" % summary([r["walk_r3"] for r in runs[name]]))
            print("  parity gate frames checked: %s" % runs[name][-1]["parity"])
            if name != libs[0][0]:
                print("  dump byte-identical with %s: %s" % (libs[0][0], same_tree(os.path.join(tmp, "dump_" + libs[0][0]), os.path.join(tmp, "dump_" + name))))
    shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
