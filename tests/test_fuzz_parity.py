"""Randomised differential test: seeded random scenarios (topology, latency law, loss, fault
injections between runs, host sends, scheduled client traffic, sizing near the limits) executed on
the oracle and on the engine's kernel sources under the CPU SIMT emulator; journals must be
identical.  `MS_FUZZ_SEEDS=a:b` widens the seed range (the committed default is a handful); `MS_FUZZ_ORIGIN=1`
starts every random, heavy and sharded scenario at a counter origin near a 32-bit boundary (fuzz_origin)."""
import os

import numpy as np
import pytest

import contextlib

import emul_lib
import oracle_lib as O
from scenarios import assert_same_journal, both, compact_total, make_pair, oracle_gossip_sends


def backend():
    """MS_FUZZ_BACKEND=cuda runs the single-GPU modes on the product library of the GPU box (profiles/ has the
    log of such a run); the default is the kernel sources under the CPU SIMT emulator."""
    if os.environ.get("MS_FUZZ_BACKEND") == "cuda":
        return contextlib.nullcontext()
    return emul_lib.use()


def compact_expectation(workload, topology, latency_mean_ms, p_loss, loss_phase=False):
    """How much server -> server gossip a drawn scenario must carry in compact records (DESIGN.md 3.1):
    "eq" all of it, "le" at most all of it, "zero" none.  The fast path needs broadcast, constant latency 0,
    no loss roll, no removed endpoint, no message sent on a server's behalf (the fuzzer sends none of these
    two) and at most 4 neighbors for windows that are not block-ordered."""
    if workload != "broadcast" or topology == "total" or latency_mean_ms > 0:
        return "zero"
    if p_loss > 0 or loss_phase or topology == "tree4":
        return "le"
    return "eq"


def assert_gossip_accounting(rings, o, expect, rings0=None):
    """rings: Sim.ring_counters() of every shard; o: the oracle after the same scenario; rings0: the counters
    before it (a ring origin), else they started at 0."""
    ev, bd = o.journal()
    want = oracle_gossip_sends(ev, bd, o.n_nodes)
    if rings0 is None:
        got = sum(compact_total(rc) for rc in rings)
    else:                                                     # claims since the start, modulo 2^32
        got = sum(int((rc["ctail"] - r0["ctail"]).astype(np.uint64).sum()) for rc, r0 in zip(rings, rings0))
    if expect == "eq":
        assert got == want, (got, want)
    elif expect == "le":
        assert got <= want, (got, want)
    else:
        assert got == 0, got


def fuzz_origin(seed):
    """MS_FUZZ_ORIGIN=1: a counter origin (Sim.set_origin) drawn per seed -- message id just below 2^31 or 2^32,
    event id just below 2^32, round just below 2^15, 2^31 or 2^32, ring counters just below 2^32 with a stride,
    or all of them -- so that the scenario crosses the boundary; None otherwise."""
    if os.environ.get("MS_FUZZ_ORIGIN") != "1":
        return None
    r = np.random.default_rng(31000 + seed)
    pick = int(r.integers(6))
    o = {}
    if pick in (0, 5):
        o["msg_id"] = (1 << int(r.choice([31, 32]))) - int(r.integers(1, 3000))
    if pick in (1, 5):
        o["event_id"] = (1 << 32) - int(r.integers(1, 6000))
    if pick in (2, 5):
        o["round"] = (1 << int(r.choice([15, 31, 32]))) - int(r.integers(1, 60))
    if pick in (3, 4, 5):
        o["ring_pos"] = (1 << 32) - int(r.integers(1, 400))
        o["ring_stride"] = int(r.integers(0, 9))
    return o


def apply_origin(origin, *sims):
    """Sets `origin` on every sim; returns the engines' ring counters right after (None without an origin)."""
    if not origin:
        return None
    for s in sims:
        s.set_origin(**origin)
    return [s.ring_counters() for s in sims if hasattr(s, "ring_counters")]


def seeds():
    spec = os.environ.get("MS_FUZZ_SEEDS", "0:6")
    a, b = (int(x) for x in spec.split(":"))
    return list(range(a, b))


def random_ops(rng, n_nodes, clients, services, workload, t0_ms, n_ticks, per_tick, mids):
    rows = np.zeros(n_ticks * per_tick, dtype=O.OP_DTYPE)
    k = 0
    for t in range(n_ticks):
        for _ in range(per_tick):
            r = rows[k]
            k += 1
            c = int(rng.integers(len(clients)))
            mids[c] += 1
            r["time_ns"] = (t0_ms + t) * 1_000_000
            r["src"] = clients[c]
            b = r["body"]
            b["flags"] = O.F_MSG_ID if rng.integers(8) else 0
            b["msg_id"] = mids[c]
            if services and rng.integers(4) == 0:
                name = list(services)[int(rng.integers(len(services)))]
                r["dest"] = services[name]
                if name == "lin-tso":
                    b["type"] = O.T["ts"]
                else:
                    kind = int(rng.integers(3))
                    b["type"] = (O.T["read"], O.T["write"], O.T["cas"])[kind]
                    b["p0"] = int(rng.integers(5))
                    b["p1"] = int(rng.integers(4)) | ((int(rng.integers(4)) << 32) if kind == 2 else 0)
                    if kind == 2 and rng.integers(2):
                        b["flags"] |= O.F_CREATE
                continue
            r["dest"] = int(rng.integers(n_nodes))
            x = int(rng.integers(10))
            if workload == "broadcast":
                if x < 7:
                    b["type"] = O.T["broadcast"]
                    b["p0"] = int(rng.integers(48))           # duplicates on purpose
                elif x < 9:
                    b["type"] = O.T["read"]
                else:
                    b["type"] = O.T["topology"] if rng.integers(2) else O.T["add"]      # add: error 10
            elif workload == "g-set":
                if x < 6:
                    b["type"] = O.T["add"]
                    b["p0"] = int(rng.integers(200))
                elif x < 9:
                    b["type"] = O.T["read"]
                else:
                    b["type"] = O.T["replicate_one"]
                    b["p0"] = int(rng.integers(200))
            elif workload == "txn-list-append":
                b["type"] = O.T["txn"] if x < 9 else O.T["read"]                        # read: error 10
                b["p1"] = int(rng.integers(1 << 20))
                if x < 6:
                    b["flags"] |= O.F_APPENDS
            else:                                             # echo
                b["type"] = O.T["echo"] if x < 9 else O.T["read"]
                b["p0"], b["p1"] = int(rng.integers(1000)), int(rng.integers(1 << 40))
    return rows


@pytest.mark.parametrize("seed", seeds())
def test_random_scenario(seed):
    rng = np.random.default_rng(1000 + seed)
    workload = ("broadcast", "broadcast", "g-set", "echo", "txn-list-append")[int(rng.integers(5))]
    n = int(rng.integers(1, 40))
    topo = ("grid", "line", "total", "tree2", "tree3", "tree4")[int(rng.integers(6))]
    if topo == "total":
        n = min(n, 10)                                        # n^2 messages per value: keep inside the wheel slots
    dist = ("constant", "constant", "uniform", "exponential")[int(rng.integers(4))]
    mean = 0 if dist == "constant" and rng.integers(2) else int(rng.integers(1, 6))
    kw = dict(topology=topo, latency_dist=dist, latency_mean_ms=mean, n_values=256,
              p_loss=float(rng.choice([0.0, 0.0, 0.05, 0.3])), seed=int(rng.integers(1 << 40)))
    if workload == "g-set":
        kw["gset_interval_ms"] = int(rng.integers(3, 15))
    sizing = dict(max_endpoints=n + 24, ring_cap=1024, max_window=1024, journal_cap_log2=int(rng.integers(14, 19)),
                  calendar_slots=1024, calendar_cap=4096)
    with_services = bool(rng.integers(2)) or workload == "txn-list-append"     # txn nodes need lin-kv
    n_clients = int(rng.integers(1, 5))
    phases = int(rng.integers(2, 5))
    plan = [(int(rng.integers(6)), int(rng.integers(2, 7)), int(rng.integers(1, 12))) for _ in range(phases)]
    fault_args = rng.integers(0, 1 << 30, size=(phases, 4))

    def scenario(s, body):
        services = {}
        if with_services:
            for name in ("lin-kv", "seq-kv", "lww-kv", "lin-tso"):
                services[name] = s.add_endpoint(name, O.KIND_SERVICE)
        clients = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT if i else O.KIND_CLIENT) for i in range(n_clients)]
        if workload == "g-set":
            for i in range(n):
                s.send(clients[0], i, body("init", msg_id=9000 + i))
        r2 = np.random.default_rng(seed)                   # the same stream for both executions
        state = {"slow": False}
        mids = [0] * n_clients
        t_ms = 0
        for ph, (fault, ticks, per_tick) in enumerate(plan):
            a = [int(v) for v in fault_args[ph]]
            if fault == 1 and n > 1:
                s.drop(a[0] % n, a[1] % n)
            elif fault == 2:
                comp = [(a[0] >> (i % 30)) & 1 for i in range(n)]
                s.partition(comp)
            elif fault == 3:
                s.heal()
            elif fault == 4:                                # one level of slow! at most: x100 leaves the wheel
                if state["slow"]:
                    s.fast()
                elif dist != "exponential":
                    s.slow()
                state["slow"] = not state["slow"] if (state["slow"] or dist != "exponential") else False
            elif fault == 5:
                s.set_loss((a[0] % 40) / 100.0)
            s.schedule(random_ops(r2, n, clients, services, workload, t_ms, ticks, per_tick, mids))
            s.send(clients[0], a[2] % n, body("read", msg_id=5000 + ph))
            t_ms += ticks
            s.run(t_ms * 1_000_000)
        s.heal()
        s.run((t_ms + 40) * 1_000_000)
        got = []
        while True:                                         # what the host-visible client saw, in order
            m = s.recv(clients[0], 0)
            if m is None:
                break
            got.append((int(m["id"]), int(m["type"]), int(m["src"]), int(m["in_reply_to"]), int(m["p0"]), int(m["p1"])))
        return got, s.client_replies()

    with backend():
        g, o = make_pair(n, workload=workload, **kw, **sizing)
        rings0 = apply_origin(fuzz_origin(seed), g, o)
        rg, ro = both(g, o, scenario)
        assert rg == ro
        loss_phase = any(fault == 5 and int(fault_args[ph][0]) % 40 for ph, (fault, _, _) in enumerate(plan))
        assert_gossip_accounting([g.ring_counters()], o, compact_expectation(workload, topo, mean, kw["p_loss"], loss_phase),
                                 rings0)
        assert_same_journal(g, o)


def heavy_seeds():
    spec = os.environ.get("MS_FUZZ_HEAVY_SEEDS", "0:2")
    a, b = (int(x) for x in spec.split(":"))
    return list(range(a, b))


@pytest.mark.parametrize("seed", heavy_seeds())
def test_random_heavy_broadcast(seed):
    # the measured path under load: hundreds of values per tick, windows spanning the size classes,
    # sender-block ordering with its verify / bitonic fallbacks, per-neighbor block claims
    rng = np.random.default_rng(5000 + seed)
    n = int(rng.integers(30, 260))
    topo = ("grid", "grid", "line", "tree2", "tree4")[int(rng.integers(5))]
    mean = int(rng.choice([0, 0, 1, 2]))
    n_clients = int(rng.integers(1, 6))
    ticks = int(rng.integers(2, 6))
    per_tick = int(rng.integers(20, 400))
    max_window = int(rng.choice([1024, 2048, 4096]))
    if rng.integers(3) == 0:                                  # burst: few nodes, windows of thousands (classes 2-3)
        n, per_tick, ticks, max_window = int(rng.integers(9, 50)), int(rng.integers(800, 3000)), 2, 4096
    kw = dict(topology=topo, latency_dist="constant", latency_mean_ms=mean, n_values=ticks * per_tick + 64,
              p_loss=float(rng.choice([0.0, 0.0, 0.02])), seed=int(rng.integers(1 << 40)))
    sizing = dict(max_endpoints=n + 16, ring_cap=8192, max_window=max_window, journal_cap_log2=21,
                  calendar_slots=64, calendar_cap=1 << 16, journal_level=int(rng.choice([1, 2])))

    def scenario(s, body):
        clients = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(n_clients)]
        r2 = np.random.default_rng(seed)
        rows = np.zeros(ticks * per_tick, dtype=O.OP_DTYPE)
        hot = int(r2.integers(n))
        for k in range(len(rows)):
            r = rows[k]
            r["time_ns"] = (k // per_tick) * 1_000_000
            r["src"] = clients[int(r2.integers(n_clients))]
            r["dest"] = hot if r2.integers(4) == 0 else int(r2.integers(n))     # a hot node: big windows
            b = r["body"]
            b["type"] = O.T["broadcast"]
            b["flags"] = O.F_MSG_ID
            b["msg_id"] = k + 1
            b["p0"] = k if r2.integers(10) else int(r2.integers(max(k, 1)))       # some duplicates
        s.schedule(rows)
        s.run((ticks + 2) * 1_000_000)
        if mean:
            s.run((ticks + 2 + 600 * mean) * 1_000_000)

    with backend():
        import maelstrom_b200 as mb
        g, o = make_pair(n, workload="broadcast", **kw, **sizing)
        rings0 = apply_origin(fuzz_origin(5000 + seed), g, o)
        try:
            both(g, o, scenario)
        except mb.SimError as e:                              # the random load does not fit this sizing
            if "max_window" in str(e) or "ring overflow" in str(e) or "timing wheel" in str(e):
                pytest.skip("capacity: %s" % e)
            raise
        assert_gossip_accounting([g.ring_counters()], o, compact_expectation("broadcast", topo, mean, kw["p_loss"]), rings0)
        if sizing["journal_level"] == 2:
            assert_same_journal(g, o)
        else:
            ev_g, _ = g.drain(bodies=False)
            ev_o, _ = o.journal()
            assert len(ev_g) == len(ev_o)
            for f in ("event_id", "time_ns", "msg_id", "src", "dest"):
                assert np.array_equal(ev_g[f], ev_o[f]), f
            assert g.stats() == o.stats()
        c = g.counters()
        assert c["max_window"] <= max_window


def sharded_seeds():
    spec = os.environ.get("MS_FUZZ_SHARDED_SEEDS", "0:1")
    a, b = (int(x) for x in spec.split(":"))
    return list(range(a, b))


@pytest.mark.parametrize("seed", sharded_seeds())
def test_random_sharded(seed):
    # 2-4 emulated shards (one host thread each) against the oracle: owner map, peer-ring claims,
    # barriers, k_commit over all shards' tables, workload state read across shards
    from test_emul_sharded import check_against_oracle, run_sharded_scenario
    rng = np.random.default_rng(9000 + seed)
    world = int(rng.integers(2, 5))
    workload = ("broadcast", "broadcast", "g-set", "txn-list-append")[int(rng.integers(4))]
    n = int(rng.integers(world, 60))
    mean = int(rng.choice([0, 1, 3]))
    dist = "constant" if mean == 0 else ("constant", "uniform")[int(rng.integers(2))]
    kw = dict(topology=("grid", "line", "tree3")[int(rng.integers(3))], latency_dist=dist, latency_mean_ms=mean,
              n_values=1024, p_loss=float(rng.choice([0.0, 0.03])), seed=int(rng.integers(1 << 40)))
    if workload == "g-set":
        kw["gset_interval_ms"] = int(rng.integers(4, 12))
    n_clients = int(rng.integers(1, 5))
    ticks, per_tick = int(rng.integers(3, 10)), int(rng.integers(5, 60))
    rings, rings0 = {}, {}
    origin = fuzz_origin(9000 + seed)

    def scenario(s, body):
        if origin:
            s.set_origin(**origin)
            if hasattr(s, "ring_counters"):
                rings0[s.cfg.shard_id] = s.ring_counters()
        services = {}
        if workload == "txn-list-append" or rng_services:
            for name in ("lin-kv", "seq-kv", "lin-tso"):
                services[name] = s.add_endpoint(name, O.KIND_SERVICE)
        clients = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(n_clients)]
        if workload == "g-set":
            for i in range(n):
                s.send(clients[0], i, body("init", msg_id=9000 + i))
        r2 = np.random.default_rng(seed)
        s.schedule(random_ops(r2, n, clients, services, workload, 0, ticks, per_tick, [0] * n_clients))
        s.run((ticks + 30 + 12 * mean) * 1_000_000)
        if hasattr(s, "ring_counters"):
            rings[s.cfg.shard_id] = s.ring_counters()     # (one entry per shard thread)

    rng_services = bool(rng.integers(2))
    wl = {"broadcast": O.W_BROADCAST, "g-set": O.W_GSET, "txn-list-append": O.W_TXN}[workload]
    ev, st, now, rnd = run_sharded_scenario(
        world, n, dict(workload=workload, ring_cap=2048, max_window=1024, journal_cap_log2=20, max_endpoints=n + 24,
                       calendar_slots=256, calendar_cap=8192, **kw), scenario)
    o = O.Sim(n, workload=wl, **kw)
    check_against_oracle(o, scenario, ev, st, now, rnd)
    assert len(rings) == world
    assert_gossip_accounting([rings[r] for r in range(world)], o, compact_expectation(workload, kw["topology"], mean, kw["p_loss"]),
                             [rings0[r] for r in range(world)] if origin else None)


def raft_seeds():
    spec = os.environ.get("MS_FUZZ_RAFT_SEEDS", "0:0")        # slow (seconds of virtual time): off by default
    a, b = (int(x) for x in spec.split(":"))
    return list(range(a, b))


@pytest.mark.parametrize("seed", raft_seeds())
def test_random_raft(seed):
    # elections under loss / latency / partitions that come and go, client traffic through every node
    rng = np.random.default_rng(7000 + seed)
    n = int(rng.integers(2, 8))
    mean = int(rng.choice([0, 1, 4]))
    kw = dict(latency_dist="constant" if mean == 0 else ("constant", "exponential")[int(rng.integers(2))],
              latency_mean_ms=mean, p_loss=float(rng.choice([0.0, 0.02, 0.15])), seed=int(rng.integers(1 << 40)))
    n_clients = 3
    phases = [(int(rng.integers(4)), int(rng.integers(300, 2600))) for _ in range(int(rng.integers(3, 6)))]
    masks = rng.integers(1, 1 << 16, size=len(phases))

    def scenario(s, body):
        clients = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(n_clients)]
        for i in range(n):
            s.send(clients[0], i, body("init", msg_id=9000 + i))
        r2 = np.random.default_rng(seed)
        t_ms, mid = 0, 0
        for (fault, dur), mask in zip(phases, masks):
            if fault == 1:
                s.partition([(int(mask) >> i) & 1 for i in range(n)])
            elif fault == 2:
                s.heal()
            elif fault == 3 and n > 1:
                s.drop(int(mask) % n, (int(mask) >> 4) % n)
            rows = np.zeros(int(r2.integers(0, 40)), dtype=O.OP_DTYPE)
            for k in range(len(rows)):
                r = rows[k]
                mid += 1
                r["time_ns"] = (t_ms + int(r2.integers(dur))) * 1_000_000
                r["src"] = clients[int(r2.integers(n_clients))]
                r["dest"] = int(r2.integers(n))
                b = r["body"]
                b["flags"] = O.F_MSG_ID
                b["msg_id"] = mid
                b["p0"] = int(r2.integers(4))
                kind = int(r2.integers(3))
                b["type"] = (O.T["read"], O.T["write"], O.T["cas"])[kind]
                b["p1"] = int(r2.integers(4)) | ((int(r2.integers(4)) << 32) if kind == 2 else 0)
            rows = rows[np.argsort(rows["time_ns"], kind="stable")]
            s.schedule(rows)
            t_ms += dur
            s.run(t_ms * 1_000_000)
        return [s.raft_state(i) for i in range(n)], s.client_replies()

    with backend():
        g, o = make_pair(n, workload="lin-kv", max_endpoints=n + 8, ring_cap=1024, max_window=512,
                         journal_cap_log2=19, calendar_slots=256, calendar_cap=4096, **kw)
        rg, ro = both(g, o, scenario)
        assert rg == ro
        assert_same_journal(g, o)
