#!/usr/bin/env python
"""Partition nemesis on the device (ms_set_nemesis) against the same schedule driven from the host, on one GPU.  The
two sides alternate (device, host, device, host, ...) in one process, with the idle-time jump on in both:

  device  Sim.nemesis(...): k_nemesis applies every cluster's ops inside the round loop;
  host    the run stops at every instant of the schedule (taken from the first device run's nemesis records) and
          installs the composed component vector with ms_net_partition: one host sync, one upload of the vector and
          the end of any idle-time jump per instant.  A majorities-ring start becomes one drop! per cut pair; an
          instant with a ring stop heals, then re-installs the vector and the drops of every cluster still in a ring.

Per side it prints, after every virtual second, the progress so far, and at the end the wall seconds of the timed
ms_run calls, rounds executed and jumped, kernel launches, host stops and a sha256 digest of the journal events, the
client history (nemesis records left out) and the final node states.  The digests of the two sides must be equal.

    python tools/bench_nemesis.py [--reps 2] [--seconds 10] [--interval-ms 2000] [--targets 0] [--latency-ms 0]
                                  [--out FILE]

--targets is ms_nemesis_config.targets (0 = one, majority and minority-third; 0x17 adds majorities-ring).
--latency-ms is the constant message latency.  With the ring at latency 0 this shape stops advancing virtual time
1.905 s after the nemesis starts (DESIGN.md 6.2); run the ring at --latency-ms 1.

Scenario: 819 five-node Raft clusters with 8190 lin-kv clients (the scale of tests/test_nemesis.py), elections done,
then `--seconds` of virtual time under one partition schedule per cluster; the clients stop invoking two seconds
before the end."""
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
from maelstrom_b200.engine import H_NEMESIS, HF_NEM_STOP, HF_NEM_MAJORITIES_RING, KIND_SIM_CLIENT  # noqa: E402
from maelstrom_b200._lib import OP_DTYPE  # noqa: E402

MS = 1_000_000
N, G, CLIENTS = 4095, 5, 8190
T0 = 4500 * MS
SEED = 0x4D41454C
SIM = dict(workload="lin-kv", latency_dist="constant", latency_mean_ms=0, raft_group=G, journal_level=1,
           server_ring_cap=64, server_max_window=32, rpc_table=64, n_keys=16, raft_log_cap=512, journal_cap_log2=24,
           ring_cap=64, max_window=32, seed=SEED)


def setup(s, seconds):
    c = s.add_endpoint("c99999", KIND_SIM_CLIENT)
    a = np.zeros(N, dtype=OP_DTYPE)
    for i in range(N):
        a[i]["time_ns"], a[i]["src"], a[i]["dest"] = i // 32 * MS, c, i
        a[i]["body"]["type"] = mb.body("init").type
        a[i]["body"]["flags"] = mb.body("init", msg_id=1).flags
        a[i]["body"]["msg_id"] = 1 + i
    s.schedule(a)
    s.run(T0)
    s.add_kv_clients(CLIENTS, interval_ns=1000 * MS, time_limit_ns=T0 + (seconds - 2) * 1000 * MS,
                     key_period_ns=500 * MS, keys_per_group=8)


def host_plan(records):
    """[(instant, [(cluster, op, f), ...])] in (cluster, op) order, from a device run's nemesis records"""
    plan = {}
    for r in records:
        plan.setdefault(int(r["time_ns"]), []).append((int(r["value"]), int(r["op"]), int(r["f"])))
    return sorted(plan.items())


def ring_cuts(c, j):
    """the (src, dest) server pairs that ring start j of cluster c cuts"""
    pos = mb.nemesis_grudge(SEED, c, G, j, HF_NEM_MAJORITIES_RING).astype(np.int64)
    m = G // 2 + 1
    dest, src = np.nonzero(((pos[None, :] - pos[:, None] + m // 2) % G) >= m)
    return [(c * G + int(a), c * G + int(b)) for a, b in zip(src, dest)]


def run_once(device, seconds, interval_ns, targets, latency_ms, plan):
    s = mb.Sim(N, max_endpoints=N + CLIENTS + 8, **dict(SIM, latency_mean_ms=latency_ms))
    s.idle_jump()
    setup(s, seconds)                                 # untimed: elections / initialisation
    until = T0 + seconds * 1000 * MS
    c0 = s.counters()
    r0 = s.round
    d = hashlib.sha256()
    n_events, n_cli, stops, drops, heals = 0, 0, 0, 0, 0
    ring = {}                                         # host side: cluster -> the cut pairs of its ring
    nem = []
    vec = np.full(N, 0xFFFFFFFF, dtype=np.uint32)
    todo = list(plan or [])
    wall = 0.0
    if device:
        s.nemesis(time_limit_ns=until, interval_ns=interval_ns, start_ns=T0, targets=targets)
    for k in range(1, seconds + 1):
        stretch = T0 + k * 1000 * MS
        t0 = time.perf_counter()
        if not device:
            while todo and todo[0][0] < stretch:
                t, group = todo.pop(0)
                s.run(t)
                reinstall, new = False, []
                for c, j, f in group:
                    if f == HF_NEM_STOP and c in ring:
                        del ring[c]
                        reinstall = True
                    elif f == HF_NEM_MAJORITIES_RING:
                        ring[c] = ring_cuts(c, j)
                        new.append(c)
                    else:
                        vec[c * G:(c + 1) * G] = 0xFFFFFFFF if f == HF_NEM_STOP else 2 * c + mb.nemesis_grudge(SEED, c, G, j, f)
                if reinstall:
                    s.heal()
                    heals += 1
                    new = list(ring)
                s.partition(vec)
                for c in new:
                    for src, dest in ring.get(c, ()):
                        s.drop(src, dest)
                        drops += 1
                stops += 1
        s.run(stretch)                                # Sim.run drains the journal whenever the device asks
        h = s.history()
        wall += time.perf_counter() - t0
        ev, _ = s.drain(bodies=False)                 # untimed: the digest
        d.update(np.ascontiguousarray(ev).tobytes())
        cli = h[h["client"] != H_NEMESIS]
        d.update(np.ascontiguousarray(cli).tobytes())
        nem.append(h[h["client"] == H_NEMESIS])
        n_events += len(ev)
        n_cli += len(cli)
        print("  %s t=%ds wall=%.2fs rounds=%d executed=%d" % ("device" if device else "host", k, wall, s.round - r0,
                                                            s.counters()["rounds"] - c0["rounds"]), flush=True)
    d.update(json.dumps([[s.raft_state(i) for i in range(0, N, 7)], s.stats(), s.now, s.round]).encode())
    c1 = s.counters()
    nem = np.concatenate(nem)
    ran = c1["rounds"] - c0["rounds"]
    out = dict(side="device" if device else "host", wall_s=wall, virtual_s=seconds, rounds=s.round - r0,
               rounds_executed=ran, rounds_jumped=s.round - r0 - ran, launches=c1["launches"] - c0["launches"],
               host_stops=stops, host_drops=drops, host_heals=heals, nemesis_records=int(len(nem)), clusters_with_records=int(len(set(nem["value"].tolist()))),
               client_records=n_cli, events=n_events, partition_drops=c1["partition_drops"] - c0["partition_drops"],
               digest=d.hexdigest()[:32])
    s.close()
    return out, nem


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--seconds", type=int, default=10)
    ap.add_argument("--interval-ms", type=int, default=2000)
    ap.add_argument("--targets", type=lambda x: int(x, 0), default=0)
    ap.add_argument("--latency-ms", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"gpu": gpu_info(), "scenario": dict(clusters=N // G, servers_per_cluster=G, clients=CLIENTS,
                                               virtual_s=a.seconds, interval_ms=a.interval_ms, targets=a.targets,
                                               latency_ms=a.latency_ms),
           "runs": []}
    plan = None
    for rep in range(a.reps):
        for device in (True, False):
            r, nem = run_once(device, a.seconds, a.interval_ms * MS, a.targets, a.latency_ms, plan)
            if device and plan is None:
                plan = host_plan(nem)
            res["runs"].append(r)
            print(json.dumps(r), flush=True)
    dev = [r for r in res["runs"] if r["side"] == "device"]
    host = [r for r in res["runs"] if r["side"] == "host"]
    assert len({r["digest"] for r in res["runs"]}) == 1, "outputs differ between the device and the host-driven nemesis"
    res["digest_equal"] = True
    res["speedup_median"] = float(np.median([x["wall_s"] for x in host]) / np.median([x["wall_s"] for x in dev]))
    res["gpu_after"] = gpu_info()
    print(json.dumps(res), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
