"""Sharded engine under the CPU SIMT emulator (tests/native/emul): G shards of ONE process, one
host thread per shard, mapping each other's rings through the emulator's pointer-carrying IPC
handles.  Exercises the multi-shard kernel paths (owner map, peer-ring claims, k_barrier,
k_commit over all shards' tables) without GPUs; the merged journal must equal the oracle's and
therefore the single-shard journal.  The GPU twin is tests/test_gpu_sharded.py."""
import ctypes as C
import threading

import numpy as np
import pytest

import emul_lib
import oracle_lib as O
from scenarios import random_broadcast_ops


def run_sharded(world, n, per_tick, latency_ms, until_ns, n_ticks=3, seed=17, **kw):
    from maelstrom_b200 import _lib
    from maelstrom_b200.engine import KIND_SIM_CLIENT, Sim
    from maelstrom_b200.sharded import merge_journals
    n_values = n_ticks * per_tick + 8
    blobs = [None] * world
    out = [None] * world
    errs = []
    sync = threading.Barrier(world)
    ops_box = {}

    def shard(rank):
        try:
            g = Sim(n, workload="broadcast", topology="grid", n_values=n_values, ring_cap=4096, max_window=2048,
                    journal_cap_log2=20, max_endpoints=n + 8, latency_dist="constant",
                    latency_mean_ms=latency_ms, journal_level=1, n_shards=world, shard_id=rank, **kw)
            blob = (C.c_ubyte * _lib.SHARD_BLOB_BYTES)()
            g._chk(g.L.ms_shard_handles(g.h, blob))
            blobs[rank] = bytes(blob)
            sync.wait()
            for peer in range(world):
                buf = (C.c_ubyte * _lib.SHARD_BLOB_BYTES).from_buffer_copy(blobs[peer])
                g._chk(g.L.ms_shard_connect(g.h, peer, buf))
            sync.wait()
            cs = [g.add_endpoint("c%d" % i, KIND_SIM_CLIENT) for i in range(3)]
            ops, _ = random_broadcast_ops(n, cs, n_ticks=n_ticks, per_tick=per_tick, seed=seed)
            ops_box[rank] = ops
            g.schedule(ops)
            g.run(until_ns)
            ev, _ = g.drain(bodies=False)
            out[rank] = (ev, g.stats(), g.now, g.round)
            sync.wait()          # nobody frees rings a peer may still be writing to
            g.close()
        except Exception as e:   # noqa: BLE001
            errs.append((rank, repr(e)))
            sync.abort()

    with emul_lib.use():
        ts = [threading.Thread(target=shard, args=(r,)) for r in range(world)]
        for t in ts:
            t.start()
        for t in ts:
            t.join(timeout=600)
    assert not errs, errs
    merged = merge_journals([o[0] for o in out])
    stats = {}
    for _, st, _, _ in out:
        for c, d in st.items():
            for k, v in d.items():
                stats.setdefault(c, {}).setdefault(k, 0)
                stats[c][k] += v
    assert len({(o[2], o[3]) for o in out}) == 1      # every shard ends at the same time and round
    return merged, stats, out[0][2], out[0][3], ops_box[0]


@pytest.mark.parametrize("world,n,per_tick,latency_ms", [(2, 64, 120, 0), (4, 64, 60, 0), (3, 100, 40, 2)])
def test_emulated_shards_equal_oracle(world, n, per_tick, latency_ms):
    until = 30_000_000 if latency_ms else 4_000_000
    ev, st, now, rnd, ops = run_sharded(world, n, per_tick, latency_ms, until)
    o = O.Sim(n, workload=O.W_BROADCAST, topology="grid", n_values=3 * per_tick + 8,
              latency_dist="constant", latency_mean_ms=latency_ms)
    for i in range(3):
        o.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT)
    o.schedule(ops)
    o.run(until)
    ev_o, _ = o.journal()
    assert len(ev) == len(ev_o), (len(ev), len(ev_o))
    for f in ("event_id", "time_ns", "msg_id", "src", "dest"):
        assert np.array_equal(ev[f], ev_o[f]), f
    assert st == o.stats()
    assert now == o.now and rnd == o.round


def run_sharded_scenario(world, n, sim_kw, scenario):
    """scenario(sim, body) runs identically on every shard (one host thread each); returns the
    merged level-1 journal, summed stats and the common (now, round)."""
    from maelstrom_b200 import _lib, body
    from maelstrom_b200.engine import Sim
    from maelstrom_b200.sharded import merge_journals
    blobs, out, errs = [None] * world, [None] * world, []
    sync = threading.Barrier(world)

    def shard(rank):
        try:
            g = Sim(n, journal_level=1, n_shards=world, shard_id=rank, **sim_kw)
            blob = (C.c_ubyte * _lib.SHARD_BLOB_BYTES)()
            g._chk(g.L.ms_shard_handles(g.h, blob))
            blobs[rank] = bytes(blob)
            sync.wait()
            for peer in range(world):
                buf = (C.c_ubyte * _lib.SHARD_BLOB_BYTES).from_buffer_copy(blobs[peer])
                g._chk(g.L.ms_shard_connect(g.h, peer, buf))
            sync.wait()
            scenario(g, body)
            ev, _ = g.drain(bodies=False)
            out[rank] = (ev, g.stats(), g.now, g.round)
            sync.wait()
            g.close()
        except Exception:   # noqa: BLE001
            import traceback
            errs.append((rank, traceback.format_exc()))
            sync.abort()

    with emul_lib.use():
        ts = [threading.Thread(target=shard, args=(r,)) for r in range(world)]
        for t in ts:
            t.start()
        for t in ts:
            t.join(timeout=600)
    assert not errs, errs
    stats = {}
    for _, st, _, _ in out:
        for c, d in st.items():
            for k, v in d.items():
                stats.setdefault(c, {}).setdefault(k, 0)
                stats[c][k] += v
    assert len({(o[2], o[3]) for o in out}) == 1
    return merge_journals([o[0] for o in out]), stats, out[0][2], out[0][3]


def check_against_oracle(o, scenario, ev, st, now, rnd):
    scenario(o, O.body)
    ev_o, _ = o.journal()
    assert len(ev) == len(ev_o), (len(ev), len(ev_o))
    for f in ("event_id", "time_ns", "msg_id", "src", "dest"):
        assert np.array_equal(ev[f], ev_o[f]), f
    assert st == o.stats()
    assert now == o.now and rnd == o.round


@pytest.mark.parametrize("world,dist,mean", [(2, "constant", 0), (3, "uniform", 3)])
def test_emulated_shards_gset_and_services(world, dist, mean):
    # g-set nodes merge snapshots that live on other shards; service endpoints live on whichever
    # shard owns them; sim clients talk to both
    from test_workload_gset import scheduled_adds_and_reads
    from test_workload_services import SVC, random_service_ops
    n = 12
    kw = dict(n_values=512, gset_interval_ms=9, latency_dist=dist, latency_mean_ms=mean)

    def scenario(s, body):
        sv = {name: s.add_endpoint(name, O.KIND_SERVICE) for name in SVC}
        cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(4)]
        for i in range(n):
            s.send(cs[0], i, body("init", msg_id=1000 + i))
        a, _ = scheduled_adds_and_reads(n, 4, n_ticks=25, per_tick=4, seed=8)
        a["src"] = a["src"] - n + cs[0]                 # the helper assumes clients start at index n
        b = random_service_ops(4, cs[0], sv, n_ticks=25, per_tick=6, seed=9)
        ops = np.concatenate([a, b])
        ops = ops[np.argsort(ops["time_ns"], kind="stable")]
        s.schedule(ops)
        s.run(60_000_000)

    ev, st, now, rnd = run_sharded_scenario(
        world, n, dict(workload="g-set", ring_cap=512, max_window=512, journal_cap_log2=20, max_endpoints=n + 16, **kw),
        scenario)
    o = O.Sim(n, workload=O.W_GSET, **kw)
    check_against_oracle(o, scenario, ev, st, now, rnd)


@pytest.mark.parametrize("world", [2, 3])
def test_emulated_shards_txn_list_append(world):
    # txn nodes on different shards race for the root held by the lin-kv service on yet another one
    n = 5
    kw = dict(latency_dist="uniform", latency_mean_ms=2, p_loss=0.05)

    def scenario(s, body):
        s.add_endpoint("lin-kv", O.KIND_SERVICE)
        cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(5)]
        rng = np.random.default_rng(31)
        rows = np.zeros(240, dtype=O.OP_DTYPE)
        for k in range(240):
            r = rows[k]
            r["time_ns"] = (k // 4) * 1_000_000
            r["src"] = cs[k % 5]
            r["dest"] = int(rng.integers(n))
            b = r["body"]
            b["type"] = O.T["txn"]
            b["flags"] = O.F_MSG_ID | (O.F_APPENDS if rng.integers(3) else 0)
            b["msg_id"] = k + 1
            b["p1"] = 1000 + k
        s.schedule(rows)
        s.run(110_000_000)

    ev, st, now, rnd = run_sharded_scenario(
        world, n, dict(workload="txn-list-append", ring_cap=256, max_window=256, journal_cap_log2=18,
                       max_endpoints=n + 16, **kw), scenario)
    check_against_oracle(O.Sim(n, workload=O.W_TXN, **kw), scenario, ev, st, now, rnd)


def test_emulated_shards_raft():
    # a 5-node Raft cluster over 2 shards: votes and append_entries cross shards, followers copy
    # entries out of the leader shard's payload heap
    n = 5
    kw = dict(latency_dist="constant", latency_mean_ms=1)

    def scenario(s, body):
        cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(3)]
        for i in range(n):
            s.send(cs[0], i, body("init", msg_id=900 + i))
        rng = np.random.default_rng(41)
        rows = np.zeros(90, dtype=O.OP_DTYPE)
        for k in range(90):
            r = rows[k]
            r["time_ns"] = 4_300_000_000 + (k // 2) * 1_000_000
            r["src"] = cs[k % 3]
            r["dest"] = int(rng.integers(n))
            b = r["body"]
            b["flags"] = O.F_MSG_ID
            b["msg_id"] = k + 1
            b["p0"] = int(rng.integers(3))
            kind = int(rng.integers(3))
            b["type"] = (O.T["read"], O.T["write"], O.T["cas"])[kind]
            b["p1"] = int(rng.integers(3)) | ((int(rng.integers(3)) << 32) if kind == 2 else 0)
        s.schedule(rows)
        s.run(4_600_000_000)

    ev, st, now, rnd = run_sharded_scenario(
        2, n, dict(workload="lin-kv", ring_cap=256, max_window=256, journal_cap_log2=18, max_endpoints=n + 16, **kw),
        scenario)
    check_against_oracle(O.Sim(n, workload=O.W_RAFT, **kw), scenario, ev, st, now, rnd)
    assert st["servers"]["send-count"] > 30 and st["clients"]["recv-count"] > 150


@pytest.mark.parametrize("world,fmt,latency", [(2, 8, 0), (3, 32, 0), (2, 8, 2)])
def test_emulated_shards_stream_their_journal(world, fmt, latency):
    # ms_run_streamed on every shard: each hands over only its own endpoints' events, with their event
    # ids (MS_JFMT_16 / MS_JFMT_EVENT); all shards keep taking the same back-pressure decisions; the
    # union over the shards is the oracle's journal
    n = 36
    kw = dict(n_values=2048, latency_dist="constant", latency_mean_ms=latency)
    got = {}
    lock = threading.Lock()

    def scenario(s, body):
        cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(3)]
        ops, _ = random_broadcast_ops(n, cs, n_ticks=20, per_tick=12, seed=23)
        s.schedule(ops)
        if hasattr(s, "run_streamed"):
            mine = []

            def sink(info, rounds, ev):
                assert info["range_events"] >= info["n_events"] and info["format"] in (16, 32)
                mine.append(ev.copy())

            s.run_streamed((25 + 80 * latency) * 1_000_000, sink, fmt=fmt, buf_events=1500, decode=True)
            with lock:
                got[s.cfg.shard_id] = np.concatenate(mine) if mine else np.zeros(0, dtype=O.EVENT_DTYPE)
        else:
            s.run((25 + 80 * latency) * 1_000_000)

    ev_left, st, now, rnd = run_sharded_scenario(
        world, n, dict(workload="broadcast", topology="grid", ring_cap=1024, max_window=512, journal_cap_log2=16,
                       max_endpoints=n + 8, **kw), scenario)
    assert len(ev_left) == 0                                     # everything went out through the streams
    o = O.Sim(n, workload=O.W_BROADCAST, topology="grid", **kw)
    scenario(o, O.body)
    ev_o, _ = o.journal()
    allv = np.concatenate([got[r] for r in range(world)])
    assert len(allv) == len(ev_o) > 4000
    order = np.argsort(allv["event_id"] & np.uint64((1 << 63) - 1), kind="stable")
    merged = allv[order]
    for f in ("event_id", "time_ns", "msg_id", "src", "dest"):
        assert np.array_equal(merged[f], ev_o[f]), f
    assert all(len(got[r]) > 0 for r in range(world))
    assert st == o.stats() and now == o.now and rnd == o.round


def test_emulated_shards_discarded_journal_adaptive_batches():
    # journal_discard + no mailbox endpoints: ms_run sizes its batches of rounds from the previous call (also on
    # shards, where every shard must take the same decision or the barriers would not pair up); state vs the oracle
    world, n = 3, 30
    kw = dict(topology="grid", n_values=512, seed=77)

    def scenario(s, body):
        cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(3)]
        ops, _ = random_broadcast_ops(n, cs, n_ticks=20, per_tick=6, seed=12)
        s.schedule(ops)
        for t in (5, 10, 15, 20, 24):
            s.run(t * 1_000_000)

    ev, st, now, rnd = run_sharded_scenario(world, n, dict(workload="broadcast", ring_cap=512, max_window=256, journal_discard=1,
                                                            max_endpoints=n + 8, **kw), scenario)
    o = O.Sim(n, workload=O.W_BROADCAST, **kw)
    scenario(o, O.body)
    assert len(ev) == 0 and st == o.stats() and now == o.now and rnd == o.round
    assert st["servers"]["recv-count"] > 5000


@pytest.mark.parametrize("glue", [True, False], ids=["glue", "no_glue"])
@pytest.mark.parametrize("world", [2, 3, 4])
def test_emulated_shards_claim_peer_compact_rings(world, glue, monkeypatch):
    # an 8 x 8 grid whose rows are split across the shards: gossip over a row boundary claims compact ring space
    # on a peer shard.  Every shard reports its own servers' ring counters; together they must be the single-shard
    # run's, and the compact records the oracle's server -> server broadcast sends.  MS_NO_GLUE=1 takes the
    # k_snapshot launch instead of k_glue between rounds.
    from maelstrom_b200.sharded import shard_owner
    from scenarios import compact_total, oracle_gossip_sends
    if not glue:
        monkeypatch.setenv("MS_NO_GLUE", "1")
    n = 64
    kw = dict(topology="grid", n_values=1024, seed=29)
    counters = {}
    lock = threading.Lock()

    def scenario(s, body):
        cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(3)]
        ops, _ = random_broadcast_ops(n, cs, n_ticks=6, per_tick=20, seed=33)
        s.schedule(ops)
        s.run(3_000_000)
        s.run(12_000_000)
        if hasattr(s, "ring_counters") and s.cfg.n_shards > 1:
            with lock:
                counters[s.cfg.shard_id] = s.ring_counters()

    sim_kw = dict(workload="broadcast", ring_cap=1024, max_window=512, journal_cap_log2=19, max_endpoints=n + 8, **kw)
    ev, st, now, rnd = run_sharded_scenario(world, n, sim_kw, scenario)
    o = O.Sim(n, workload=O.W_BROADCAST, **kw)
    check_against_oracle(o, scenario, ev, st, now, rnd)
    ev_o, bd_o = o.journal()
    from maelstrom_b200.engine import Sim
    with emul_lib.use():
        one = Sim(n, journal_level=1, **sim_kw)
        scenario(one, None)
        single = one.ring_counters()
        one.close()
    owners = np.array([shard_owner(e, n, world) for e in range(n)])
    assert len(set(owners.tolist())) == world
    for k, v in single.items():
        summed = sum(counters[r][k].astype(np.uint64) for r in range(world))
        assert np.array_equal(summed, v.astype(np.uint64)), k
        for r in range(world):                          # a shard reports only the servers it owns
            assert not counters[r][k][owners != r].any(), (k, r)
    assert compact_total(single) == oracle_gossip_sends(ev_o, bd_o, n) > 1000


def test_emulated_eight_shards_broadcast_glue_path():
    # the shard count of the driver's scaling run: 8 shards, no timing wheel -> one k_glue launch between rounds
    world, n = 8, 64
    kw = dict(topology="grid", n_values=512, seed=5)

    def scenario(s, body):
        cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(4)]
        ops, _ = random_broadcast_ops(n, cs, n_ticks=6, per_tick=12, seed=21)
        s.schedule(ops)
        s.run(4_000_000)
        s.run(9_000_000)

    ev, st, now, rnd = run_sharded_scenario(world, n, dict(workload="broadcast", ring_cap=1024, max_window=512, journal_cap_log2=19,
                                                            max_endpoints=n + 8, **kw), scenario)
    check_against_oracle(O.Sim(n, workload=O.W_BROADCAST, **kw), scenario, ev, st, now, rnd)
    assert len(ev) > 20000
