#!/usr/bin/env python3
"""Class-2 occupancy sweep: broadcast-flood throughput against the number of 2048-slot round-kernel CTAs per SM.

    python tools/occupancy_sweep.py [--runs 4] [--out FILE] [--build-only] [-- extra bench.py arguments]

The product library fits 4 class-2 CTAs (256 threads, 64 registers, 51 KB of dynamic and 4 KB of static shared memory)
on an H100 SM.  The variants are the same sources built with -DMS_CLS2_SMEM_PAD=<bytes>: every class-2 launch asks
for that much more dynamic shared memory, so only 3 or 2 of its CTAs fit, and the engine sizes class 2's persistent
grid from the same query.  Nothing else changes, so the slope from 2 to 4 CTAs/SM says what more class-2 windows in
flight would buy.  Each library's CTAs/SM is read back from cudaOccupancyMaxActiveBlocksPerMultiprocessor
(msk_round_occupancy), then the three libraries run bench.py alternating (tools/ab_bench.py's runner), --runs each.

--build-only (re)compiles the product library and the variants and exits (no GPU needed); without it, only missing
libraries are built, so build again after changing the sources.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import __graft_entry__ as G  # noqa: E402
import ab_bench  # noqa: E402

# Per-CTA footprint on an SM = dynamic + static (4064 B) + 1 KB the hardware reserves; an SM offers 228 KB.
# Unpadded: 51 232 + 4 064 + 1 024 = 56 320 B -> 4 fit.  +16 384 -> 72 704 B -> 3 fit.  +45 056 -> 101 376 B -> 2 fit.
VARIANTS = (("cls2pad3", 16384, 3), ("cls2pad2", 45056, 2))
CLS2_CAP, CLS2_THREADS = 2048, 256


def build_all(force):
    if force or not os.path.exists(G.SO):
        G.build(force=force)
    libs = [("base", G.SO, 0, 4)]
    for name, pad, expect in VARIANTS:
        path = os.path.join(ROOT, "maelstrom_b200", "libmaelstrom_b200_%s.so" % name)
        if force or not os.path.exists(path):
            print("building %s (MS_CLS2_SMEM_PAD=%d)" % (name, pad), flush=True)
            G.build_variant(name, ["MS_CLS2_SMEM_PAD=%d" % pad])
        libs.append((name, path, pad, expect))
    return libs


def cls2_ctas_per_sm(path):
    lib = ctypes.CDLL(path, mode=ctypes.RTLD_LOCAL)
    lib.msk_round_smem_bytes.restype = ctypes.c_size_t
    lib.msk_round_smem_bytes.argtypes = [ctypes.c_uint32]
    lib.msk_round_smem_attr.argtypes = [ctypes.c_size_t]
    lib.msk_round_occupancy.argtypes = [ctypes.c_int, ctypes.c_size_t]
    smem = lib.msk_round_smem_bytes(CLS2_CAP)
    if lib.msk_round_smem_attr(smem) != 0:
        raise RuntimeError("cudaFuncSetAttribute failed for %s" % path)
    return smem, lib.msk_round_occupancy(CLS2_THREADS, smem)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=4)
    ap.add_argument("--out", default="", help="write the summary as JSON lines")
    ap.add_argument("--build-only", action="store_true")
    ap.add_argument("extra", nargs="*", help="passed on to bench.py (after --)")
    args = ap.parse_args()
    if args.runs < 4:
        ap.error("--runs must be at least 4")
    libs = build_all(args.build_only)
    if args.build_only:
        return
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True, check=True).stdout.strip()
    print("gpu: " + gpu)
    occ = {}
    for name, path, pad, expect in libs:
        smem, nb = cls2_ctas_per_sm(path)
        occ[name] = nb
        print("%-9s pad %6d  class-2 dynamic smem %6d B  CTAs/SM %d (expected %d)" % (name, pad, smem, nb, expect))
        if nb != expect:
            sys.exit("%s: class 2 fits %d CTAs/SM, not %d" % (name, nb, expect))

    rows = {name: [] for name, _, _, _ in libs}
    for k in range(args.runs):
        for name, path, _, _ in libs:
            r = ab_bench.run_bench(path, ["--no-e2e", "--no-cpu"] + args.extra)
            rows[name].append(r)
            print("%-9s[%d] value %.6g  ms_per_step %.4f  avg_launch_us %.2f  clocks %s" %
                  (name, k, r["value"], r["ms_per_step"], r["roofline"]["avg_launch_us"], json.dumps(r["clocks"])),
                  flush=True)

    base_med = statistics.median(r["value"] for r in rows["base"])
    out = []
    for name, path, pad, _ in libs:
        rs = rows[name]
        v = [r["value"] for r in rs]
        ms = [r["ms_per_step"] for r in rs]
        us = [r["roofline"]["avg_launch_us"] for r in rs]
        rec = {"lib": name, "cls2_smem_pad": pad, "cls2_ctas_per_sm": occ[name], "gpu": gpu, "runs": len(rs),
               "value_median": statistics.median(v), "value_min": min(v), "value_max": max(v),
               "ms_per_step_median": statistics.median(ms), "avg_launch_us_median": statistics.median(us),
               "value_vs_base": statistics.median(v) / base_med,
               "clock_reasons": sorted({str(x) for r in rs for x in r["clocks"].get("reasons", [])})}
        out.append(rec)
        print("%-9s CTAs/SM %d  value median %.4g [%.4g, %.4g]  ms/tick %.3f  us/launch %.1f  vs base %.4f" %
              (name, occ[name], rec["value_median"], rec["value_min"], rec["value_max"], rec["ms_per_step_median"],
               rec["avg_launch_us_median"], rec["value_vs_base"]))
    by = {r["cls2_ctas_per_sm"]: r["value_median"] for r in out}
    if 3 in by and 4 in by:
        print("3 -> 4 class-2 CTAs/SM: %+.1f %% throughput" % (100.0 * (by[4] / by[3] - 1.0)))
    if 2 in by and 3 in by:
        print("2 -> 3 class-2 CTAs/SM: %+.1f %% throughput" % (100.0 * (by[3] / by[2] - 1.0)))
    if args.out:
        with open(args.out, "w") as f:
            for rec in out:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
