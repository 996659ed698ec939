#!/usr/bin/env python3
"""A/B of two engine libraries on one GPU, in one process tree, alternating.

    python tools/ab_bench.py A.so B.so [--runs 4] [--dump DIR] [-- extra bench.py arguments]

Runs `bench.py --no-e2e --no-cpu` with MS_B200_LIB=A, then B, then A, ... (`--runs` each, at least 4), prints every
run's value, ms_per_step, roofline.avg_launch_us and clocks block, then the median and min-max of each side and
whether the two ranges overlap.  With --dump it also runs each side once with `--dump-outputs` (end-to-end arm
included: the journal sample comes from it) and compares every .npy byte for byte.

A is the baseline: build it from the parent commit into a git-ignored path before comparing (e.g. a worktree's
`python -c "import __graft_entry__ as g; g.build()"`, then copy its libmaelstrom_b200.so aside).
"""
import argparse
import filecmp
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BENCH = os.path.join(ROOT, "bench.py")


def run_bench(lib, extra):
    env = dict(os.environ, MS_B200_LIB=os.path.abspath(lib))
    out = subprocess.run([sys.executable, BENCH] + extra, env=env, cwd=ROOT, check=True,
                         stdout=subprocess.PIPE, text=True).stdout
    lines = [l for l in out.splitlines() if l.startswith("{")]
    return json.loads(lines[-1])


def summary(name, rows):
    for key, get in (("value", lambda r: r["value"]), ("ms_per_step", lambda r: r["ms_per_step"]),
                     ("avg_launch_us", lambda r: r["roofline"]["avg_launch_us"])):
        xs = [get(r) for r in rows]
        print("%s %-14s median %.6g  min %.6g  max %.6g  (n=%d)" % (name, key, statistics.median(xs), min(xs), max(xs), len(xs)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("lib_a")
    ap.add_argument("lib_b")
    ap.add_argument("--runs", type=int, default=4)
    ap.add_argument("--dump", default="", metavar="DIR", help="also compare --dump-outputs of both sides under DIR/a, DIR/b")
    ap.add_argument("extra", nargs="*", help="passed on to bench.py (after --)")
    args = ap.parse_args()
    if args.runs < 4:
        ap.error("--runs must be at least 4")
    for lib in (args.lib_a, args.lib_b):
        if not os.path.exists(lib):
            ap.error("no such library: " + lib)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True, check=True).stdout.strip()
    print("gpu: " + gpu)

    rows = {"A": [], "B": []}
    for k in range(args.runs):
        for name, lib in (("A", args.lib_a), ("B", args.lib_b)):
            r = run_bench(lib, ["--no-e2e", "--no-cpu"] + args.extra)
            rows[name].append(r)
            print("%s[%d] value %.6g  ms_per_step %.4f  avg_launch_us %.2f  clocks %s" %
                  (name, k, r["value"], r["ms_per_step"], r["roofline"]["avg_launch_us"], json.dumps(r["clocks"])))
            sys.stdout.flush()
    summary("A", rows["A"])
    summary("B", rows["B"])
    va = [r["value"] for r in rows["A"]]
    vb = [r["value"] for r in rows["B"]]
    ma, mb = statistics.median(va), statistics.median(vb)
    print("B / A median value: %.4f   ranges overlap: %s" % (mb / ma, not (min(vb) > max(va) or min(va) > max(vb))))
    slow = [r["clocks"].get("reasons") for r in rows["A"] + rows["B"] if r["clocks"].get("reasons")]
    print("clock slowdown reasons seen: %s" % (slow if slow else "none"))

    ok = True
    if args.dump:
        dirs = {}
        for name, lib in (("a", args.lib_a), ("b", args.lib_b)):
            dirs[name] = os.path.join(os.path.abspath(args.dump), name)
            os.makedirs(dirs[name], exist_ok=True)
            run_bench(lib, ["--no-cpu", "--dump-outputs", dirs[name]] + args.extra)
        fa = sorted(f for f in os.listdir(dirs["a"]) if f.endswith(".npy"))
        fb = sorted(f for f in os.listdir(dirs["b"]) if f.endswith(".npy"))
        if fa != fb or not fa:
            print("dump: file lists differ: %s vs %s" % (fa, fb))
            ok = False
        for f in fa:
            same = f in fb and filecmp.cmp(os.path.join(dirs["a"], f), os.path.join(dirs["b"], f), shallow=False)
            print("dump %-28s %s" % (f, "identical" if same else "DIFFERENT"))
            ok = ok and same
        print("dump outputs byte-identical: %s" % ok)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
