#!/usr/bin/env python
"""First numbers for the node programs that are not the headline benchmark (bench.py stays the
contract for that one): g-set, services, txn-list-append and Raft on ONE GPU, each timed with the
engine's own CUDA-event timer around ms_run, journal level 0 (kernel path), inputs resident.

    python tools/bench_workloads.py                 # on the GPU
    python tools/bench_workloads.py --emul --tiny   # script check on the CPU emulator (test infra)

Prints one JSON line per workload: delivered messages per second of wall time on the device,
rounds, virtual time covered, and the algorithmic bytes the design note assigns to the workload.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def ops_array(n, dtype):
    return np.zeros(n, dtype=dtype)


def timed_run(sim, until_ns):
    sim.timer_begin()
    t0 = time.time()
    sim.run(until_ns)
    wall = time.time() - t0
    ms = sim.timer_end()
    c = sim.counters()
    return dict(device_ms=ms, wall_s=wall, rounds=c["rounds"], sends=c["sends"], recvs=c["recvs"],
                launches=c["launches"], msgs_per_s=(c["recvs"] / (ms / 1e3)) if ms > 0 else None)


def bench_gset(mb, n, interval_ms, n_values, ticks, adds_per_tick):
    from maelstrom_b200.engine import KIND_SIM_CLIENT, OP_DTYPE, TYPES, F_MSG_ID
    sim = mb.Sim(n, workload="g-set", n_values=n_values, gset_interval_ms=interval_ms, journal_level=0,
                 latency_dist="exponential", latency_mean_ms=5, ring_cap=max(1024, 2 * n), max_window=max(1024, 2 * n),
                 max_endpoints=n + 8, calendar_slots=256, calendar_cap=max(1 << 16, 8 * n * n // 16))
    c = sim.add_endpoint("c0", KIND_SIM_CLIENT)
    rows = ops_array(n + ticks * adds_per_tick, OP_DTYPE)
    for i in range(n):
        rows[i]["src"], rows[i]["dest"] = c, i
        rows[i]["body"]["type"], rows[i]["body"]["flags"], rows[i]["body"]["msg_id"] = TYPES["init"], F_MSG_ID, i + 1
    rng = np.random.default_rng(1)
    k = n
    for t in range(ticks):
        for _ in range(adds_per_tick):
            r = rows[k]
            k += 1
            r["time_ns"] = (1 + t) * 1_000_000
            r["src"], r["dest"] = c, int(rng.integers(n))
            r["body"]["type"], r["body"]["flags"], r["body"]["msg_id"] = TYPES["add"], F_MSG_ID, k
            r["body"]["p0"] = int(rng.integers(n_values))
    sim.schedule(rows)
    out = timed_run(sim, (ticks + 3 * interval_ms + 60) * 1_000_000)
    out.update(workload="g-set", nodes=n, interval_ms=interval_ms,
               algorithmic_bytes_per_replicate_full=272 + 4 * ((n_values + 31) // 32))
    return out


def bench_services(mb, per_tick, ticks):
    from maelstrom_b200.engine import KIND_SERVICE, KIND_SIM_CLIENT, OP_DTYPE, TYPES, F_MSG_ID
    sim = mb.Sim(1, workload="echo", journal_level=0, ring_cap=1 << 15, max_window=1 << 13, max_endpoints=64)
    sv = [sim.add_endpoint(name, KIND_SERVICE) for name in ("lin-kv", "seq-kv", "lww-kv", "lin-tso")]
    cs = [sim.add_endpoint("c%d" % i, KIND_SIM_CLIENT) for i in range(16)]
    rng = np.random.default_rng(2)
    rows = ops_array(per_tick * ticks, OP_DTYPE)
    rows["time_ns"] = (np.arange(len(rows)) // per_tick) * 1_000_000
    rows["src"] = np.asarray(cs)[rng.integers(len(cs), size=len(rows))]
    which = rng.integers(4, size=len(rows))
    rows["dest"] = np.asarray(sv)[which]
    kind = rng.integers(3, size=len(rows))
    rows["body"]["type"] = np.where(which == 3, TYPES["ts"], np.asarray([TYPES["read"], TYPES["write"], TYPES["cas"]])[kind])
    rows["body"]["flags"] = F_MSG_ID
    rows["body"]["msg_id"] = np.arange(len(rows)) + 1
    rows["body"]["p0"] = rng.integers(1024, size=len(rows))
    rows["body"]["p1"] = rng.integers(16, size=len(rows)) | (rng.integers(16, size=len(rows)) << 32)
    sim.schedule(rows)
    out = timed_run(sim, (ticks + 2) * 1_000_000)
    out.update(workload="services", requests_per_tick=per_tick, algorithmic_bytes_per_request=2 * 272)
    return out


def bench_txn(mb, n, per_tick, ticks):
    from maelstrom_b200.engine import KIND_SERVICE, KIND_SIM_CLIENT, OP_DTYPE, TYPES, F_MSG_ID, F_APPENDS
    sim = mb.Sim(n, workload="txn-list-append", journal_level=0, ring_cap=1 << 15, max_window=1 << 13,
                 max_endpoints=n + 32)
    sim.add_endpoint("lin-kv", KIND_SERVICE)
    cs = [sim.add_endpoint("c%d" % i, KIND_SIM_CLIENT) for i in range(16)]
    rng = np.random.default_rng(3)
    rows = ops_array(per_tick * ticks, OP_DTYPE)
    rows["time_ns"] = (np.arange(len(rows)) // per_tick) * 1_000_000
    rows["src"] = np.asarray(cs)[rng.integers(len(cs), size=len(rows))]
    rows["dest"] = rng.integers(n, size=len(rows))
    rows["body"]["type"] = TYPES["txn"]
    rows["body"]["flags"] = F_MSG_ID | np.where(rng.integers(2, size=len(rows)) == 1, F_APPENDS, 0)
    rows["body"]["msg_id"] = np.arange(len(rows)) + 1
    rows["body"]["p1"] = np.arange(len(rows)) + 1
    sim.schedule(rows)
    out = timed_run(sim, (ticks + 4) * 1_000_000)
    out.update(workload="txn-list-append", nodes=n, txns_per_tick=per_tick, messages_per_txn=6)
    return out


def bench_raft(mb, n, virtual_ms, writes_per_tick):
    from maelstrom_b200.engine import KIND_SIM_CLIENT, OP_DTYPE, TYPES, F_MSG_ID
    sim = mb.Sim(n, workload="lin-kv", journal_level=0, ring_cap=1 << 12, max_window=1 << 11, max_endpoints=n + 16)
    cs = [sim.add_endpoint("c%d" % i, KIND_SIM_CLIENT) for i in range(4)]
    t0 = 4200
    n_ops = n + (virtual_ms - t0) * writes_per_tick
    rows = ops_array(n_ops, OP_DTYPE)
    for i in range(n):
        rows[i]["src"], rows[i]["dest"] = cs[0], i
        rows[i]["body"]["type"], rows[i]["body"]["flags"], rows[i]["body"]["msg_id"] = TYPES["init"], F_MSG_ID, i + 1
    rng = np.random.default_rng(4)
    k = np.arange(n, n_ops)
    rows["time_ns"][n:] = (t0 + (k - n) // writes_per_tick) * 1_000_000
    rows["src"][n:] = np.asarray(cs)[rng.integers(4, size=len(k))]
    rows["dest"][n:] = rng.integers(n, size=len(k))
    rows["body"]["type"][n:] = np.asarray([TYPES["read"], TYPES["write"]])[rng.integers(2, size=len(k))]
    rows["body"]["flags"][n:] = F_MSG_ID
    rows["body"]["msg_id"][n:] = k + 1
    rows["body"]["p0"][n:] = rng.integers(64, size=len(k))
    rows["body"]["p1"][n:] = rng.integers(1000, size=len(k))
    sim.schedule(rows)
    out = timed_run(sim, virtual_ms * 1_000_000)
    out.update(workload="lin-kv (Raft)", nodes=n, virtual_ms=virtual_ms, leader=[i for i in range(n) if sim.raft_state(i)["state"] == 3])
    return out


def card():
    """name and power limit of the GPU, read next to the measurement they belong to"""
    import subprocess
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def bench_kv_clients(mb, n, group, steps, step_ms=200, interval_ms=1000):
    """BASELINE config 4's shape closed loop: clusters of `group` Raft nodes, 2 lin-kv clients per node on the
    device (ms_add_kv_clients), the partition nemesis of bench.py --config raft64k (random halves at every even
    virtual second, healed at every odd one; the default 12 steps after the warm-up step see one such cycle).  The history is drained after every step, as a checker's feed
    would; device time is the engine's CUDA-event timer around each step's rounds."""
    from maelstrom_b200.engine import KIND_SIM_CLIENT, OP_DTYPE, TYPES, F_MSG_ID
    n_clients = (2 * n) // (2 * group) * (2 * group)
    sim = mb.Sim(n, workload="lin-kv", latency_dist="constant", latency_mean_ms=0, journal_level=0,
                 max_endpoints=n + n_clients + 8, ring_cap=256, max_window=128, server_ring_cap=64, server_max_window=32,
                 raft_group=group, rpc_table=64, n_keys=16, raft_log_cap=2048)
    c = sim.add_endpoint("c%d" % n_clients, KIND_SIM_CLIENT)
    rows = ops_array(n, OP_DTYPE)
    rows["src"], rows["dest"] = c, np.arange(n)
    rows["time_ns"] = np.arange(n) // 128 * 1_000_000   # the sink's inbox takes 128 init_ok per round
    ramp_ms = 4600 + -(-(n // 128) // step_ms) * step_ms
    rows["body"]["type"], rows["body"]["flags"], rows["body"]["msg_id"] = TYPES["init"], F_MSG_ID, np.arange(n) + 1
    sim.schedule(rows)
    sim.run(ramp_ms * 1_000_000)                       # the first elections happen 2-4 s after init (raft.py:249-251)
    sim.add_kv_clients(n_clients, interval_ns=interval_ms * 1_000_000, time_limit_ns=1 << 62,
                       key_period_ns=1_000_000_000, keys_per_group=16)
    rng = np.random.default_rng(0x4D41454C)
    tally = np.zeros(4, dtype=np.int64)                # invoke / ok / fail / info
    dev_ms = wall = 0.0
    m0 = r0 = 0
    for k in range(steps + 1):                         # step 0 is the warm-up: not timed, not counted
        now_ms = ramp_ms + k * step_ms
        if now_ms % 1000 == 0:
            if (now_ms // 1000) % 2 == 0:
                sim.partition(rng.integers(0, 2, size=n).astype(np.uint32))
            else:
                sim.heal()
        t0 = time.time()
        sim.timer_begin()
        sim.run((now_ms + step_ms) * 1_000_000)
        ms = sim.timer_end()                           # ends in a synchronise on the event
        h = sim.history()
        dt = time.time() - t0
        if k == 0:
            m0, r0 = sim.stats()["all"]["msg-count"], sim.counters()["recvs"]
            continue
        dev_ms += ms
        wall += dt
        tally += np.bincount(h["type"], minlength=4)[:4]
    msgs = sim.stats()["all"]["msg-count"] - m0
    recvs = sim.counters()["recvs"] - r0
    done = int(tally[1:].sum())
    return dict(workload="lin-kv (Raft), closed-loop clients on the device", nodes=n, cluster_size=group,
                clients=n_clients, virtual_ms=steps * step_ms, client_interval_ms=interval_ms, latency="constant 0 ms",
                nemesis="random halves for 1 s, healed for 1 s", device_ms=dev_ms, wall_s=wall, rounds=sim.counters()["rounds"],
                ops_invoked=int(tally[0]), ops_completed=done, ok=int(tally[1]), fail=int(tally[2]), info=int(tally[3]),
                ops_per_s_wall=done / wall if wall > 0 else None,
                msgs_per_s=recvs / (dev_ms / 1e3) if dev_ms > 0 else None,
                msgs_per_op=msgs / int(tally[0]) if tally[0] else None, card=card())


def bench_kv_proxy(mb, n, group, steps, service="lin-kv", step_ms=200, interval_ms=100):
    """The GPU scale shape of tests/test_kv_proxy.py: n lin-kv proxies (demo/ruby/lin_kv_proxy.rb) over one kv service,
    2 closed-loop lin-kv clients per node (ms_add_kv_clients, groups of 2 x `group`).  Every request passes through the
    one service endpoint, whose window is walked by one thread: that window is the serial hot spot.  The history is
    drained after every step; device time is the engine's CUDA-event timer around each step's rounds."""
    from maelstrom_b200.engine import KIND_SERVICE, KIND_SIM_CLIENT, OP_DTYPE, TYPES, F_MSG_ID
    n_clients = (2 * n) // (2 * group) * (2 * group)
    window = 1 << max(n_clients - 1, 1).bit_length()                 # a service window takes every client's request
    sim = mb.Sim(n, workload="lin-kv-proxy", proxy_service=service, latency_dist="constant", latency_mean_ms=0,
                 journal_level=0, max_endpoints=n + n_clients + 8, ring_cap=window, max_window=window, server_ring_cap=64,
                 server_max_window=32, raft_group=group, rpc_table=64, n_keys=n_clients // (2 * group) * 8)
    sim.add_endpoint(service, KIND_SERVICE)
    c = sim.add_endpoint("c%d" % n_clients, KIND_SIM_CLIENT)
    rows = ops_array(n, OP_DTYPE)
    rows["src"], rows["dest"] = c, np.arange(n)
    rows["body"]["type"], rows["body"]["flags"], rows["body"]["msg_id"] = TYPES["init"], F_MSG_ID, np.arange(n) + 1
    sim.schedule(rows)
    sim.run(step_ms * 1_000_000)
    sim.add_kv_clients(n_clients, interval_ns=interval_ms * 1_000_000, time_limit_ns=1 << 62,
                       key_period_ns=500_000_000, keys_per_group=8)
    tally = np.zeros(4, dtype=np.int64)                # invoke / ok / fail / info
    dev_ms = wall = 0.0
    m0 = r0 = 0
    for k in range(steps + 1):                         # step 0 is the warm-up: not timed, not counted
        now_ms = (k + 1) * step_ms
        t0 = time.time()
        sim.timer_begin()
        sim.run((now_ms + step_ms) * 1_000_000)
        ms = sim.timer_end()                           # ends in a synchronise on the event
        h = sim.history()
        dt = time.time() - t0
        if k == 0:
            m0, r0 = sim.stats()["all"]["msg-count"], sim.counters()["recvs"]
            continue
        dev_ms += ms
        wall += dt
        tally += np.bincount(h["type"], minlength=4)[:4]
    msgs = sim.stats()["all"]["msg-count"] - m0
    recvs = sim.counters()["recvs"] - r0
    done = int(tally[1:].sum())
    return dict(workload="lin-kv proxies over %s, closed-loop clients on the device" % service, nodes=n, group=group,
                clients=n_clients, virtual_ms=steps * step_ms, client_interval_ms=interval_ms, latency="constant 0 ms",
                device_ms=dev_ms, wall_s=wall, rounds=sim.counters()["rounds"], ops_invoked=int(tally[0]),
                ops_completed=done, ok=int(tally[1]), fail=int(tally[2]), info=int(tally[3]),
                ops_per_s_wall=done / wall if wall > 0 else None,
                msgs_per_s=recvs / (dev_ms / 1e3) if dev_ms > 0 else None,
                msgs_per_op=msgs / int(tally[0]) if tally[0] else None, card=card())


def bench_kafka(mb, n, clients_per_node, keys, steps, step_ms=200, interval_ms=100):
    """The GPU scale shape of tests/test_kafka.py: n single-node kafka logs (demo/clojure/kafka_single_node.clj) with
    `keys` keys each, clients_per_node closed-loop kafka clients per node (ms_add_kafka_clients, 25 % assign, 10 %
    crash, the rest send / poll).  The history is drained after every step; device time is the engine's CUDA-event
    timer around each step's rounds."""
    from maelstrom_b200.engine import KIND_SIM_CLIENT, OP_DTYPE, TYPES, F_MSG_ID
    n_clients = n * clients_per_node
    cap = max(1024, 2 * clients_per_node * (steps + 2) * step_ms // interval_ms)   # sends per key, with room
    sim = mb.Sim(n, workload="kafka", kafka_keys=keys, kafka_log_cap=cap, latency_dist="constant", latency_mean_ms=0,
                 journal_level=0, max_endpoints=n + n_clients + 8, ring_cap=64, max_window=64, server_ring_cap=64,
                 server_max_window=32)
    c = sim.add_endpoint("c%d" % (1 << 30), KIND_SIM_CLIENT)
    rows = ops_array(n, OP_DTYPE)
    rows["src"], rows["dest"] = c, np.arange(n)
    rows["body"]["type"], rows["body"]["flags"], rows["body"]["msg_id"] = TYPES["init"], F_MSG_ID, np.arange(n) + 1
    rows["time_ns"] = (np.arange(n) % 128) * 1_000_000       # 32 init_ok a millisecond fit the sink's ring
    rows = rows[np.argsort(rows["time_ns"], kind="stable")]
    sim.schedule(rows)
    sim.run(step_ms * 1_000_000)
    sim.add_kafka_clients(n_clients, interval_ns=interval_ms * 1_000_000, time_limit_ns=1 << 62, assign_permille=250,
                          crash_permille=100)
    tally = np.zeros(4, dtype=np.int64)                # invoke / ok / fail / info
    dev_ms = wall = 0.0
    m0 = r0 = 0
    for k in range(steps + 1):                         # step 0 is the warm-up: not timed, not counted
        now_ms = (k + 1) * step_ms
        t0 = time.time()
        sim.timer_begin()
        sim.run((now_ms + step_ms) * 1_000_000)
        ms = sim.timer_end()                           # ends in a synchronise on the event
        h = sim.kafka_history()
        dt = time.time() - t0
        if k == 0:
            m0, r0 = sim.stats()["all"]["msg-count"], sim.counters()["recvs"]
            continue
        dev_ms += ms
        wall += dt
        tally += np.bincount(h["type"], minlength=4)[:4]
    msgs = sim.stats()["all"]["msg-count"] - m0
    recvs = sim.counters()["recvs"] - r0
    done = int(tally[1:].sum())
    return dict(workload="single-node kafka logs, closed-loop kafka clients on the device", nodes=n, keys=keys,
                clients=n_clients, virtual_ms=steps * step_ms, client_interval_ms=interval_ms, latency="constant 0 ms",
                device_ms=dev_ms, wall_s=wall, rounds=sim.counters()["rounds"], ops_invoked=int(tally[0]),
                ops_completed=done, ok=int(tally[1]), fail=int(tally[2]), info=int(tally[3]),
                ops_per_s_wall=done / wall if wall > 0 else None,
                msgs_per_s=recvs / (dev_ms / 1e3) if dev_ms > 0 else None,
                msgs_per_op=msgs / int(tally[0]) if tally[0] else None, card=card())


def bench_pn_counter(mb, n, group, clients_per_node, steps, step_ms=200, interval_ms=100, replicate_ms=1000):
    """The GPU scale shape of tests/test_counters.py: n PN-counter nodes (demo/ruby/pn_counter.rb) in blocks of
    `group`, replicating every replicate_ms, with clients_per_node closed-loop counter clients per node
    (ms_add_gen_clients, half adds, half reads).  The history is drained after every step; device time is the engine's
    CUDA-event timer around each step's rounds."""
    from maelstrom_b200.engine import KIND_SIM_CLIENT, OP_DTYPE, TYPES, F_MSG_ID
    n_clients = n * clients_per_node
    sim = mb.Sim(n, workload="pn-counter", raft_group=group, gset_interval_ms=replicate_ms, latency_dist="constant",
                 latency_mean_ms=0, journal_level=0, max_endpoints=n + n_clients + 8, ring_cap=64, max_window=64,
                 server_ring_cap=64, server_max_window=32)
    c = sim.add_endpoint("c%d" % (1 << 30), KIND_SIM_CLIENT)
    rows = ops_array(n, OP_DTYPE)
    rows["src"], rows["dest"] = c, np.arange(n)
    rows["body"]["type"], rows["body"]["flags"], rows["body"]["msg_id"] = TYPES["init"], F_MSG_ID, np.arange(n) + 1
    rows["time_ns"] = (np.arange(n) % 128) * 1_000_000       # 32 init_ok a millisecond fit the sink's ring
    rows = rows[np.argsort(rows["time_ns"], kind="stable")]
    sim.schedule(rows)
    sim.run(step_ms * 1_000_000)
    sim.add_gen_clients(n_clients, interval_ns=interval_ms * 1_000_000, time_limit_ns=1 << 62)
    tally = np.zeros(4, dtype=np.int64)                # invoke / ok / fail / info
    dev_ms = wall = 0.0
    m0 = r0 = 0
    for k in range(steps + 1):                         # step 0 is the warm-up: not timed, not counted
        now_ms = (k + 1) * step_ms
        t0 = time.time()
        sim.timer_begin()
        sim.run((now_ms + step_ms) * 1_000_000)
        ms = sim.timer_end()                           # ends in a synchronise on the event
        h = sim.history()
        dt = time.time() - t0
        if k == 0:
            m0, r0 = sim.stats()["all"]["msg-count"], sim.counters()["recvs"]
            continue
        dev_ms += ms
        wall += dt
        tally += np.bincount(h["type"], minlength=4)[:4]
    msgs = sim.stats()["all"]["msg-count"] - m0
    recvs = sim.counters()["recvs"] - r0
    done = int(tally[1:].sum())
    return dict(workload="PN-counter CRDT nodes, closed-loop counter clients on the device", nodes=n, group=group,
                clients=n_clients, virtual_ms=steps * step_ms, client_interval_ms=interval_ms,
                replicate_ms=replicate_ms, latency="constant 0 ms", device_ms=dev_ms, wall_s=wall,
                rounds=sim.counters()["rounds"], ops_invoked=int(tally[0]), ops_completed=done, ok=int(tally[1]),
                fail=int(tally[2]), info=int(tally[3]), ops_per_s_wall=done / wall if wall > 0 else None,
                msgs_per_s=recvs / (dev_ms / 1e3) if dev_ms > 0 else None,
                msgs_per_op=msgs / int(tally[0]) if tally[0] else None, card=card())


def bench_txn_rw(mb, n, group, clients_per_node, steps, step_ms=200, interval_ms=100, key_count=4):
    """The GPU scale shape of tests/test_txn_rw.py: n txn-rw-register nodes (demo/clojure/txn_rw_register_hat.clj) in
    blocks of `group`, replicating every 100 ms, with clients_per_node closed-loop txn clients per node
    (ms_add_txn_rw_clients, 1 to 4 micro-ops, key_count keys at a time).  The history is drained after every step;
    device time is the engine's CUDA-event timer around each step's rounds."""
    from maelstrom_b200.engine import KIND_SIM_CLIENT, OP_DTYPE, TYPES, F_MSG_ID
    n_clients = n * clients_per_node
    cap = 2 * (steps + 2) * step_ms * clients_per_node // interval_ms + 64   # ~2 txns a client per interval at most
    sim = mb.Sim(n, workload="txn-rw-register", raft_group=group, txn_rw_log_cap=cap, latency_dist="constant",
                 latency_mean_ms=0, journal_level=0, max_endpoints=n + n_clients + 8, ring_cap=64, max_window=64,
                 server_ring_cap=64, server_max_window=32)
    c = sim.add_endpoint("c%d" % (1 << 30), KIND_SIM_CLIENT)
    rows = ops_array(n, OP_DTYPE)
    rows["src"], rows["dest"] = c, np.arange(n)
    rows["body"]["type"], rows["body"]["flags"], rows["body"]["msg_id"] = TYPES["init"], F_MSG_ID, np.arange(n) + 1
    rows["time_ns"] = (np.arange(n) % 128) * 1_000_000       # 32 init_ok a millisecond fit the sink's ring
    rows = rows[np.argsort(rows["time_ns"], kind="stable")]
    sim.schedule(rows)
    sim.run(step_ms * 1_000_000)
    sim.add_txn_rw_clients(n_clients, interval_ns=interval_ms * 1_000_000, time_limit_ns=1 << 62,
                           key_period_ns=500 * 1_000_000, key_count=key_count)
    tally = np.zeros(4, dtype=np.int64)                # invoke / ok / fail / info
    dev_ms = wall = 0.0
    m0 = r0 = 0
    for k in range(steps + 1):                         # step 0 is the warm-up: not timed, not counted
        now_ms = (k + 1) * step_ms
        t0 = time.time()
        sim.timer_begin()
        sim.run((now_ms + step_ms) * 1_000_000)
        ms = sim.timer_end()                           # ends in a synchronise on the event
        h = sim.txn_rw_history()
        dt = time.time() - t0
        if k == 0:
            m0, r0 = sim.stats()["all"]["msg-count"], sim.counters()["recvs"]
            continue
        dev_ms += ms
        wall += dt
        tally += np.bincount(h["type"], minlength=4)[:4]
    msgs = sim.stats()["all"]["msg-count"] - m0
    recvs = sim.counters()["recvs"] - r0
    done = int(tally[1:].sum())
    return dict(workload="txn-rw-register nodes, closed-loop txn clients on the device", nodes=n, group=group,
                clients=n_clients, virtual_ms=steps * step_ms, client_interval_ms=interval_ms, replicate_ms=100,
                key_count=key_count, latency="constant 0 ms", device_ms=dev_ms, wall_s=wall,
                rounds=sim.counters()["rounds"], ops_invoked=int(tally[0]), ops_completed=done, ok=int(tally[1]),
                fail=int(tally[2]), info=int(tally[3]), ops_per_s_wall=done / wall if wall > 0 else None,
                msgs_per_s=recvs / (dev_ms / 1e3) if dev_ms > 0 else None,
                msgs_per_op=msgs / int(tally[0]) if tally[0] else None, card=card())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="", help="run one case: g-set, services, txn, raft, kv-clients, kv-proxy, kafka, pn-counter or txn-rw-register")
    ap.add_argument("--emul", action="store_true", help="run on the CPU SIMT emulator (script check only)")
    ap.add_argument("--tiny", action="store_true")
    a = ap.parse_args()
    import maelstrom_b200 as mb
    ctx = None
    if a.emul:
        import emul_lib
        ctx = emul_lib.use()
        ctx.__enter__()
    try:
        if a.tiny:
            runs = {"g-set": lambda: bench_gset(mb, 12, 8, 512, 10, 4), "services": lambda: bench_services(mb, 40, 5),
                    "txn": lambda: bench_txn(mb, 3, 12, 5), "raft": lambda: bench_raft(mb, 3, 4260, 2),
                    "kv-clients": lambda: bench_kv_clients(mb, 11, 5, 3), "kv-proxy": lambda: bench_kv_proxy(mb, 15, 5, 3),
                    "kafka": lambda: bench_kafka(mb, 16, 4, 4, 3), "pn-counter": lambda: bench_pn_counter(mb, 15, 5, 2, 3),
                    "txn-rw-register": lambda: bench_txn_rw(mb, 16, 2, 2, 3)}
        else:
            runs = {"g-set": lambda: bench_gset(mb, 1024, 100, 1 << 14, 200, 64), "services": lambda: bench_services(mb, 1 << 14, 20),
                    "txn": lambda: bench_txn(mb, 256, 1 << 11, 20), "raft": lambda: bench_raft(mb, 5, 10_000, 4),
                    "kv-clients": lambda: bench_kv_clients(mb, 65536, 5, 12), "kv-proxy": lambda: bench_kv_proxy(mb, 4095, 5, 15),
                    "kafka": lambda: bench_kafka(mb, 4096, 4, 4, 15),
                    "pn-counter": lambda: bench_pn_counter(mb, 4095, 5, 4, 15),
                    "txn-rw-register": lambda: bench_txn_rw(mb, 4096, 2, 4, 15)}
        for name, r in runs.items():
            if not a.only or a.only == name:
                print(json.dumps(r(), sort_keys=True), flush=True)
    finally:
        if ctx:
            ctx.__exit__(None, None, None)


if __name__ == "__main__":
    main()
