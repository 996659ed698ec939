#!/usr/bin/env python
"""Idle-time jump (ms_set_idle_jump) against ticking, on one GPU: each scenario runs with the mode off and on,
alternating (off, on, off, on, ...) in one process, and prints per side the wall seconds of the timed ms_run calls,
virtual seconds per wall second, rounds executed and rounds jumped, and a sha256 digest of journal (events and
bodies) + ms_history_drain records + final node states.  The digests of the two sides must be equal.

    python tools/bench_idle.py [--reps 2] [--only raft5,broadcast25,gset16,raft4095] [--out FILE]

Scenarios: a 5-node Raft cluster with closed-loop lin-kv clients for 60 s of virtual time; 25-node broadcast with
closed-loop clients at 100 ms exponential latency; 16-node g-set at its 5 s replication interval; 819 five-node Raft
clusters with 8190 lin-kv clients (the scale of tests/test_kv_clients.py), where nearly every tick has work and the
mode only adds its two launches per round."""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import maelstrom_b200 as mb  # noqa: E402
from maelstrom_b200.engine import KIND_SIM_CLIENT  # noqa: E402
from maelstrom_b200._lib import OP_DTYPE  # noqa: E402

MS = 1_000_000


def sched(s, rows):
    a = np.zeros(len(rows), dtype=OP_DTYPE)
    for i, (t, src, dest, ty, mid, p0) in enumerate(rows):
        a[i]["time_ns"], a[i]["src"], a[i]["dest"] = t, src, dest
        a[i]["body"]["type"] = mb.body(ty).type
        a[i]["body"]["flags"] = mb.body(ty, msg_id=mid).flags
        a[i]["body"]["msg_id"], a[i]["body"]["p0"] = mid, p0
    s.schedule(a)


def raft(n, n_clients, until_ns, interval_ms, **sizing):
    def setup(s):
        c = s.add_endpoint("c99999", KIND_SIM_CLIENT)
        sched(s, [(i // 32 * MS, c, i, "init", 1 + i, 0) for i in range(n)])
        s.run(4500 * MS)
        s.add_kv_clients(n_clients, interval_ns=interval_ms * MS, time_limit_ns=until_ns - 2000 * MS,
                         key_period_ns=500 * MS, keys_per_group=8)
    args = dict(workload="lin-kv", latency_dist="constant", latency_mean_ms=0, raft_group=5, journal_level=1)
    args.update(sizing)
    return dict(n=n, sim=args, setup=setup, until=until_ns, state=lambda s: [s.raft_state(i) for i in range(0, n, 7)])


SCENARIOS = {
    "raft5": raft(5, 10, 60_000 * MS, 1000, max_endpoints=32, ring_cap=256, max_window=128, server_ring_cap=256,
                  server_max_window=128, rpc_table=256, n_keys=64, raft_log_cap=4096, journal_cap_log2=22),
    "broadcast25": dict(
        n=25, until=30_000 * MS,
        sim=dict(workload="broadcast", topology="grid", n_values=1 << 14, latency_dist="exponential", latency_mean_ms=100,
                 max_endpoints=64, ring_cap=512, max_window=256, calendar_slots=4096, calendar_cap=1 << 16, journal_level=1),
        setup=lambda s: s.add_gen_clients(10, interval_ns=1000 * MS, time_limit_ns=25_000 * MS, read_permille=500,
                                          timeout_ns=5000 * MS, quiet_ns=2000 * MS, first_name=0),
        state=lambda s: [s.node_set(k).tolist() for k in range(25)]),
    "gset16": dict(
        n=16, until=60_000 * MS,
        sim=dict(workload="g-set", latency_dist="constant", latency_mean_ms=5, n_values=1024, max_endpoints=32,
                 ring_cap=256, max_window=128, calendar_slots=64, calendar_cap=1 << 14, journal_level=1),
        setup=lambda s: sched(s, [(0, s.add_endpoint("c0", KIND_SIM_CLIENT), 0, "init", 1, 0)] +
                              [(0, 16, i, "init", i + 1, 0) for i in range(1, 16)] +
                              [(t * 1000 * MS, 16, t % 16, "add", 100 + t, t) for t in range(1, 60, 3)]),
        state=lambda s: [s.node_set(k).tolist() for k in range(16)]),
    "raft4095": raft(4095, 8190, 9000 * MS, 1000, server_ring_cap=64, server_max_window=32, rpc_table=64, n_keys=16,
                     raft_log_cap=512, journal_cap_log2=24, ring_cap=64, max_window=32, max_endpoints=4095 + 8190 + 8),
}


def run_once(name, jump):
    sc = SCENARIOS[name]
    s = mb.Sim(sc["n"], **sc["sim"])
    if jump:
        s.idle_jump()
    h = hashlib.sha256()
    sc["setup"](s)                                    # untimed: elections / initialisation
    v0, r0, x0 = s.now, s.round, s.counters()["rounds"]
    hist = []
    t0 = time.perf_counter()
    step = 1000 * MS
    while s.now < sc["until"]:
        s.run(min(s.now + step, sc["until"]))         # Sim.run drains the journal whenever the device asks
        hist.append(s.history())
    wall = time.perf_counter() - t0
    ev, bd = s.drain()
    for part in (ev, bd, np.concatenate(hist)):
        h.update(np.ascontiguousarray(part).tobytes())
    h.update(json.dumps([sc["state"](s), s.stats(), s.now, s.round]).encode())
    ran = s.counters()["rounds"] - x0
    out = dict(jump=jump, wall_s=wall, virtual_s=(s.now - v0) / 1e9, virtual_per_wall=(s.now - v0) / 1e9 / wall,
               rounds=s.round - r0, rounds_executed=ran, rounds_jumped=s.round - r0 - ran, events=int(len(ev)),
               history=int(sum(len(x) for x in hist)), digest=h.hexdigest()[:32])
    s.close()
    return out


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--only", default=",".join(SCENARIOS))
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"gpu": gpu_info(), "scenarios": {}}
    for name in a.only.split(","):
        runs = []
        for rep in range(a.reps):
            for jump in (False, True):
                r = run_once(name, jump)
                runs.append(r)
                print(name, json.dumps(r), flush=True)
        off = [r for r in runs if not r["jump"]]
        on = [r for r in runs if r["jump"]]
        assert len({r["digest"] for r in runs}) == 1, "outputs differ between the two modes"
        per_round_us = None
        if name == "raft4095":      # nearly every tick has work: the cost of the two extra launches per executed round
            per_round_us = 1e6 * (min(x["wall_s"] for x in on) - min(x["wall_s"] for x in off)) / on[0]["rounds_executed"]
        res["scenarios"][name] = dict(
            off=off, on=on, digest_equal=True,
            speedup_median=float(np.median([x["wall_s"] for x in off]) / np.median([x["wall_s"] for x in on])),
            overhead_us_per_executed_round=per_round_us)
    res["gpu_after"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
