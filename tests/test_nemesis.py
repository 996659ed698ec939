"""Partition nemesis on the device (ms_set_nemesis, DESIGN.md 2.13): one Jepsen partition schedule per cluster, run by
k_nemesis before every executed round.  The schedule is restated here from its spec with oracle_lib.philox, and each
run is compared with its host-driven twin: the same simulation without the nemesis, stopped at every restated instant
to install the composed component vector with ms_net_partition -- on the engine and on the oracle.  Journal, bodies,
statistics, node and Raft states, ms_now / ms_round and the client history must be identical; the nemesis's records
must be the restated ops.  [emul] = the kernel sources on the CPU SIMT emulator, [cuda] = an H100."""
import numpy as np
import pytest

import kv_oracle_lib as K
import oracle_lib as O
from scenarios import ops_array

pytestmark = pytest.mark.usefixtures("engine_backend")
MS = 1_000_000
NEVER = 0xFFFFFFFF
DRAW, RANK = 0x4E454D00, 0x4E454D01
ONE, MAJORITY, MINORITY_THIRD, STOP = 5, 6, 7, 8
HIST_FIELDS = ("time_ns", "order", "client", "op", "type", "f", "error", "value")
SEED = 0x4D41454C


# ----------------------------------------------------------------------------------------------- the spec, restated
def draw(seed, ctr0, ctr1, key):
    return O.philox([ctr0, ctr1, key, 0], [seed & 0xFFFFFFFF, seed >> 32])


def ceil_tick(t):
    return -(-t // MS) * MS


def schedule(seed, n_clusters, mask, interval, start, limit):
    """every op as (t_j, cluster, j, f): gen/stagger of the interval over a flip-flop of start / stop, cut at the time
    limit, with a final stop at the limit for a cluster left partitioned"""
    mask = mask or 7
    enabled = [ONE + t for t in range(3) if mask >> t & 1]
    ops = []
    for c in range(n_clusters):
        t, j, part = start, 0, False
        while True:
            x = draw(seed, j, c, DRAW)
            t += ceil_tick((x[0] * 2 * interval) >> 32)
            if t >= limit:
                break
            f = STOP if j & 1 else enabled[(x[1] * len(enabled)) >> 32]
            ops.append((t, c, j, f))
            part = f != STOP
            j += 1
        if part:
            ops.append((limit, c, j, STOP))
    return ops


def sides(seed, c, g, j, f):
    """0 = side A, 1 = side B for the servers c*g .. c*g + g - 1: ranks by (key, server) below the side's size"""
    keys = [(draw(seed, j, c * g + i, RANK)[0], i) for i in range(g)]
    m = {ONE: 1, MAJORITY: g // 2 + 1, MINORITY_THIRD: max(1, g // 3)}[f]
    out = [1] * g
    for r, (_, i) in enumerate(sorted(keys)):
        if r < m:
            out[i] = 0
    return out


def applied(ops, now0):
    """the ops grouped by the instant of the round that applies them, in (cluster, op) order"""
    by = {}
    for t, c, j, f in ops:
        by.setdefault(max(ceil_tick(t), now0), []).append((c, j, f))
    return {k: sorted(v) for k, v in sorted(by.items())}


class HostNemesis:
    """the nemesis driven from the host: run() stops at every instant of the restated schedule and installs the
    composed component vector; heal() puts every server back to never-cut as ms_net_heal does with the nemesis on"""

    def __init__(self, sim, seed, n, g, ops, now0):
        self.s, self.seed, self.g = sim, seed, g
        self.vec = np.full(n, NEVER, dtype=np.uint32)
        self.todo = list(applied(ops, now0).items())

    def run(self, until):
        while self.todo and self.todo[0][0] < until:
            t, group = self.todo.pop(0)
            self.s.run(t)
            for c, j, f in group:
                lo = c * self.g
                if f == STOP:
                    self.vec[lo:lo + self.g] = NEVER
                else:
                    sd = np.array(sides(self.seed, c, self.g, j, f), dtype=np.uint32)
                    self.vec[lo:lo + self.g] = 2 * c + sd
            self.s.partition(self.vec)
        self.s.run(until)

    def heal(self):
        self.s.heal()
        self.vec[:] = NEVER


class DeviceNemesis:
    def __init__(self, sim, **cfg):
        self.s = sim
        sim.nemesis(**cfg)

    def run(self, until):
        self.s.run(until)

    def heal(self):
        self.s.heal()


def expected_records(seed, ops, now0):
    rows = []
    for t, group in applied(ops, now0).items():
        for c, j, f in group:
            rows.append((t, NEVER, j, 3, f, 0, c))
    return rows


def nemesis_rows(h):
    m = h[h["client"] == NEVER]
    assert np.all((m["order"] & np.uint64(0xFFFFFF)) == 0xFFFFFF)
    return [(int(r["time_ns"]), int(r["client"]), int(r["op"]), int(r["type"]), int(r["f"]), int(r["error"]),
             int(r["value"])) for r in m]


def outputs(s, n, workload, hist):
    ev, bd = s.drain()
    out = {"ev": ev, "bd": bd, "stats": s.stats(), "now": s.now, "round": s.round,
           "client_replies": s.client_replies(), "undeliverable": s.undeliverable(), "hist": hist}
    if workload in ("broadcast", "g-set"):
        out["sets"] = [s.node_set(k).tolist() for k in range(n)]
    if workload == "lin-kv":
        out["raft"] = [s.raft_state(k) for k in range(n)]
    return out


def assert_same(a, b, what):
    assert len(a["ev"]) == len(b["ev"]), (what, len(a["ev"]), len(b["ev"]))
    for f in ("event_id", "time_ns", "msg_id", "src", "dest"):
        assert np.array_equal(a["ev"][f], b["ev"][f]), (what, f)
    for f in ("type", "flags", "msg_id", "in_reply_to", "p0", "p1"):
        assert np.array_equal(a["bd"][f], b["bd"][f]), (what, f)
    for k in a:
        if k not in ("ev", "bd", "hist") and k in b:
            assert a[k] == b[k], (what, k, a[k], b[k])
    assert len(a["hist"]) == len(b["hist"]), (what, len(a["hist"]), len(b["hist"]))
    for f in HIST_FIELDS:
        assert np.array_equal(a["hist"][f], b["hist"][f]), (what, f)


def twins(n, g, scenario, nem, oracle=None, jump=False, seed=SEED, **kw):
    """run A (device nemesis), run B (host-driven twin on the engine) and, if given, the oracle's host-driven run.
    scenario(sim, R) drives a simulation through R.run / R.heal and returns what it wants compared.
    Returns (A's outputs, A's nemesis rows, the restated ops)"""
    import maelstrom_b200 as mb
    workload = kw.get("workload", "broadcast")
    kw["seed"] = seed
    C = n // g
    now0 = nem.pop("now0", 0)
    cfg = dict(nem)
    ops = schedule(seed, C, cfg.get("targets", 0), cfg.get("interval_ns", 0) or 10_000 * MS, cfg.get("start_ns", 0),
                   cfg["time_limit_ns"])
    a = mb.Sim(n, **kw)
    if jump:
        a.idle_jump()
    ra = scenario(a, lambda s: DeviceNemesis(s, **cfg))
    ha = a.history()
    oa = outputs(a, n, workload, ha)
    oa["executed"] = a.counters()["rounds"]
    a.close()
    rows = nemesis_rows(ha)
    assert rows == expected_records(seed, ops, now0)
    client_a = ha[ha["client"] != NEVER]
    b = mb.Sim(n, **kw)
    rb = scenario(b, lambda s: HostNemesis(s, seed, n, g, ops, now0))
    ob = outputs(b, n, workload, b.history())
    b.close()
    assert ra == rb
    assert_same(dict(oa, hist=client_a), ob, "device nemesis vs host-driven twin")
    if oracle is not None:
        o = oracle()
        ro = scenario(o, lambda s: HostNemesis(s, seed, n, g, ops, now0))
        assert ro == ra
        ev, bd = o.journal()
        oo = {"ev": ev, "bd": bd, "stats": o.stats(), "now": o.now, "round": o.round,
              "client_replies": o.client_replies(), "undeliverable": o.undeliverable(), "hist": o.history()}
        if workload in ("broadcast", "g-set"):
            oo["sets"] = [o.node_set(k).tolist() for k in range(n)]
        if workload == "lin-kv":
            oo["raft"] = [o.raft_state(k) for k in range(n)]
        assert_same(dict(oa, hist=client_a), oo, "device nemesis vs oracle")
        o.close()
    return oa, rows, ops


# ----------------------------------------------------------------------------------------------- 1. the schedule
@pytest.mark.parametrize("seed,g,mask", [(SEED, 1, 0), (7, 2, 1), (11, 3, 2), (12, 5, 4), (99, 5, 3), (5, 64, 6)])
def test_schedule_and_grudges_match_the_restatement(seed, g, mask):
    import maelstrom_b200 as mb
    n = 3 * g if g < 64 else 64
    C = n // g
    kw = dict(workload="lin-kv", raft_group=g if g < n else 0, max_endpoints=n + 4, journal_level=0, seed=seed)
    s = mb.Sim(n, **kw)
    c = s.add_endpoint("c0", O.KIND_SIM_CLIENT)
    # interval 1 ns: every delay is 0 or 1 ns before rounding up to ticks, so half of them are zero and several ops
    # of a cluster share a round
    interval = 1
    s.nemesis(time_limit_ns=60 * MS + 300_000, interval_ns=interval, start_ns=2 * MS + 1, targets=mask)
    s.schedule(ops_array([(0, c, i, "init", 1 + i, 0) for i in range(n)]))
    seen = []
    s.run(30 * MS)
    seen.append(s.history())
    s.run(90 * MS)
    seen.append(s.history())
    h = np.concatenate(seen)
    ops = schedule(seed, C, mask, interval, 2 * MS + 1, 60 * MS + 300_000)
    assert nemesis_rows(h) == expected_records(seed, ops, 0)
    assert len(ops) > 20 * C
    times = [t for t, group in applied(ops, 0).items() for cc in set(x[0] for x in group)
             if sum(1 for x in group if x[0] == cc) > 1]
    assert times, "no round applies two ops of one cluster"
    enabled = {ONE + t for t in range(3) if (mask or 7) >> t & 1}
    fs = {f for _, _, _, f in ops if f != STOP}
    assert fs <= enabled and (len(fs) == len(enabled) or len(ops) < 40)
    assert ops[-1][0] <= 60 * MS + 300_000 and all(r[0] <= ceil_tick(60 * MS + 300_000) for r in nemesis_rows(h))
    for t, cc, j, f in ops[:40]:
        if f != STOP:
            assert mb.nemesis_grudge(seed, cc, g, j, f).tolist() == sides(seed, cc, g, j, f)
    s.close()


def test_grudge_sides_have_the_target_sizes():
    import maelstrom_b200 as mb
    for g in (1, 2, 3, 5, 64, 8192):
        for f, m in ((ONE, 1), (MAJORITY, g // 2 + 1), (MINORITY_THIRD, max(1, g // 3))):
            sd = mb.nemesis_grudge(SEED, 3, g, 4, f)
            assert int(np.count_nonzero(sd == 0)) == m
    assert mb.nemesis_grudge(SEED, 3, 5, 4, ONE).tolist() != mb.nemesis_grudge(SEED, 4, 5, 4, ONE).tolist() or \
        mb.nemesis_grudge(SEED, 3, 5, 6, ONE).tolist() != mb.nemesis_grudge(SEED, 4, 5, 6, ONE).tolist()
    with pytest.raises(mb.SimError):
        mb.nemesis_grudge(SEED, 0, 5, 0, STOP)
    with pytest.raises(mb.SimError):
        mb.nemesis_grudge(SEED, 0, 8193, 0, ONE)


# ----------------------------------------------------------------------------------------------- 2-4. twins
RAFT = dict(workload="lin-kv", latency_dist="exponential", latency_mean_ms=2, p_loss=0.02, ring_cap=256,
            max_window=128, server_ring_cap=256, server_max_window=128, raft_group=5, rpc_table=256, n_keys=64,
            raft_log_cap=2048, journal_cap_log2=20, calendar_slots=64, calendar_cap=4096)


def raft_scenario(n, n_clients, until, heal_at=None):
    def scenario(s, make):
        c = s.add_endpoint("c9999", O.KIND_SIM_CLIENT)
        s.schedule(ops_array([(i // 32 * MS, c, i, "init", 1 + i, 0) for i in range(n)]))
        s.run(3000 * MS)
        s.add_kv_clients(n_clients, interval_ns=250 * MS, time_limit_ns=until - 1500 * MS, key_period_ns=1000 * MS,
                         keys_per_group=4, timeout_ns=500 * MS)
        R = make(s)
        if heal_at:
            R.run(heal_at)
            R.heal()
        R.run(until)
        return [s.raft_state(i)["term"] for i in range(n)]
    return scenario


def raft_oracle(n, **kw):
    return lambda: K.Sim(n, workload=O.W_RAFT, latency_dist=kw["latency_dist"], latency_mean_ms=kw["latency_mean_ms"],
                         p_loss=kw.get("p_loss", 0.0), raft_group=5, rpc_table=256, seed=kw.get("seed", SEED))


@pytest.mark.parametrize("jump", [False, True])
def test_raft_clusters_with_kv_clients_under_loss(jump):
    n, n_clients = 100, 200
    until = 12_000 * MS
    nem = dict(time_limit_ns=10_000 * MS, interval_ns=800 * MS, start_ns=3200 * MS)
    kw = dict(RAFT, max_endpoints=n + n_clients + 4)
    oa, rows, ops = twins(n, 5, raft_scenario(n, n_clients, until), nem, oracle=raft_oracle(n, **kw), jump=jump, **kw)
    assert len({r[6] for r in rows}) == n // 5                      # every cluster has its own records
    assert {r[4] for r in rows} == {ONE, MAJORITY, MINORITY_THIRD, STOP}
    assert oa["stats"]["servers"]["recv-count"] > 0
    if jump:
        assert oa["executed"] < 0.9 * oa["round"]


def test_heal_mid_partition_keeps_the_schedules():
    n, n_clients = 20, 40
    until = 9000 * MS
    nem = dict(time_limit_ns=8000 * MS, interval_ns=1500 * MS, start_ns=3000 * MS, targets=2)
    kw = dict(RAFT, max_endpoints=n + n_clients + 4)
    oa, rows, ops = twins(n, 5, raft_scenario(n, n_clients, until, heal_at=5000 * MS + 1), nem,
                          oracle=raft_oracle(n, **kw), **kw)
    # some cluster was partitioned across the heal and still gets its stop afterwards
    starts = {(c, j) for t, c, j, f in ops if f != STOP and t <= 5000 * MS}
    assert any((c, j + 1) in {(cc, jj) for t, cc, jj, f in ops if t > 5000 * MS} for c, j in starts)


def broadcast_scenario(s, make):
    s.add_gen_clients(6, interval_ns=150 * MS, time_limit_ns=3000 * MS, read_permille=300, timeout_ns=500 * MS,
                      quiet_ns=500 * MS)
    R = make(s)
    R.run(1500 * MS)
    s.flaky()
    R.run(2000 * MS)
    s.set_loss(0.02)
    R.run(4500 * MS)
    return s.now


def test_broadcast_grid_with_gen_clients():
    n = 16
    kw = dict(workload="broadcast", topology="grid", n_values=1 << 10, latency_dist="exponential", latency_mean_ms=30,
              p_loss=0.02, max_endpoints=32, ring_cap=256, max_window=128, calendar_slots=256, calendar_cap=4096)
    nem = dict(time_limit_ns=3500 * MS, interval_ns=300 * MS, start_ns=100 * MS)
    oracle = lambda: O.Sim(n, workload=O.W_BROADCAST, topology="grid", n_values=1 << 10, latency_dist="exponential",
                           latency_mean_ms=30, p_loss=0.02, seed=SEED)
    oa, rows, ops = twins(n, n, broadcast_scenario, nem, oracle=oracle, **kw)
    assert len(rows) > 6 and oa["stats"]["servers"]["send-count"] > 0
    with_jump, _, _ = twins(n, n, broadcast_scenario, nem, jump=True, **kw)
    assert with_jump["executed"] < 0.9 * with_jump["round"]


def gset_scenario(s, make):
    c = s.add_endpoint("c0", O.KIND_SIM_CLIENT)
    s.schedule(ops_array([(0, c, i, "init", i + 1, 0) for i in range(6)] +
                         [(t * MS, c, t % 6, "add", 100 + t, t % 50) for t in range(5, 9000, 37)]))
    R = make(s)
    R.run(12_000 * MS)
    return [s.node_set(k).tolist() for k in range(6)]


@pytest.mark.parametrize("jump", [False, True])
def test_gset(jump):
    kw = dict(workload="g-set", latency_dist="constant", latency_mean_ms=20, n_values=64, max_endpoints=8,
              ring_cap=256, max_window=128, calendar_slots=64, calendar_cap=1024, gset_interval_ms=700)
    nem = dict(time_limit_ns=10_000 * MS, interval_ns=1000 * MS, start_ns=0, targets=5)
    oracle = lambda: O.Sim(6, workload=O.W_GSET, latency_dist="constant", latency_mean_ms=20, n_values=64,
                           gset_interval_ms=700, seed=SEED)
    oa, rows, _ = twins(6, 6, gset_scenario, nem, oracle=oracle, jump=jump, **kw)
    assert oa["stats"]["servers"]["send-count"] > 0 and len(rows) > 4
    if jump:
        assert oa["executed"] < 0.5 * oa["round"]


def txn_scenario(s, make):
    svc = s.add_endpoint("lin-kv", O.KIND_SERVICE)
    cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(3)]
    s.schedule(ops_array([(0, cs[i], i, "init", 1, 0) for i in range(3)] +
                         [(t * MS, cs[t % 3], t % 3, "txn", 10 + t, 0) for t in range(100, 6000, 90)]))
    R = make(s)
    R.run(7000 * MS)
    return svc, s.client_replies()


def test_single_key_txn_service_is_never_cut():
    kw = dict(workload="txn-list-append", max_endpoints=16, latency_dist="constant", latency_mean_ms=5)
    nem = dict(time_limit_ns=6000 * MS, interval_ns=400 * MS, start_ns=50 * MS)
    oracle = lambda: O.Sim(3, workload=O.W_TXN, latency_dist="constant", latency_mean_ms=5, seed=SEED)
    oa, rows, _ = twins(3, 3, txn_scenario, nem, oracle=oracle, **kw)
    assert oa["stats"]["servers"]["recv-count"] > 0 and len(rows) > 4


def many_clusters_scenario(n):
    def scenario(s, make):
        c = s.add_endpoint("c0", O.KIND_SIM_CLIENT)
        s.schedule(ops_array([(i // 64 * MS, c, i, "init", 1 + i, 0) for i in range(n)]))
        R = make(s)
        R.run(1600 * MS)                              # jumped: nothing acts before the first election timeouts
        R.run(2120 * MS)                              # ops in every tick while the first elections run
        return [s.raft_state(i)["term"] for i in range(n)]
    return scenario


def test_more_clusters_than_the_kernel_has_threads():
    # 560 two-node clusters: k_nemesis scans the clusters in two stretches of 512 and applies the due ops of both in
    # cluster order; the nemesis starts as the first election timeouts fire, so request_vote traffic is cut
    n = 1120
    kw = dict(workload="lin-kv", raft_group=2, max_endpoints=n + 4, ring_cap=64, max_window=64, server_ring_cap=64,
              server_max_window=64, rpc_table=64, n_keys=8, raft_log_cap=256, journal_cap_log2=22)
    nem = dict(time_limit_ns=2100 * MS, interval_ns=60 * MS, start_ns=1950 * MS)
    oa, rows, ops = twins(n, 2, many_clusters_scenario(n), nem, jump=True, **kw)
    assert len({r[6] for r in rows}) > 520 and max(r[6] for r in rows) >= 512
    # some round applies ops of clusters in both stretches
    assert any(min(x[0] for x in g) < 512 <= max(x[0] for x in g) for g in applied(ops, 0).values())
    assert oa["stats"]["servers"]["send-count"] > 0 and oa["executed"] < 0.5 * oa["round"]


def test_broadcast_cluster_larger_than_the_kernel_has_threads():
    # one cluster of 600 servers: the key and component loops of k_nemesis stride past their 512 threads
    n = 600
    kw = dict(workload="broadcast", topology="grid", n_values=64, max_endpoints=n + 4, ring_cap=64, max_window=64)

    def scenario(s, make):
        c = s.add_endpoint("c0", O.KIND_SIM_CLIENT)
        s.schedule(ops_array([(t * MS, c, (t * 97) % n, "broadcast", t + 1, t % 64) for t in range(0, 40, 3)]))
        R = make(s)
        R.run(45 * MS)
        return [len(s.node_set(k)) for k in range(0, n, 37)]
    nem = dict(time_limit_ns=40 * MS, interval_ns=2 * MS, start_ns=0)
    oa, rows, ops = twins(n, n, scenario, nem, **kw)
    assert len(rows) > 8 and {r[4] for r in rows} >= {ONE, MAJORITY, MINORITY_THIRD, STOP}
    import maelstrom_b200 as mb
    sd = mb.nemesis_grudge(SEED, 0, n, rows[0][2], rows[0][4])
    assert sd.tolist() == sides(SEED, 0, n, rows[0][2], rows[0][4])


# ----------------------------------------------------------------------------------------------- 5. edges
def test_time_limit_final_stops_and_nothing_after():
    import maelstrom_b200 as mb
    s = mb.Sim(20, workload="lin-kv", raft_group=5, max_endpoints=24, journal_level=0)
    s.nemesis(time_limit_ns=40 * MS + 500_000, interval_ns=3 * MS, start_ns=0)
    s.run(200 * MS)
    rows = nemesis_rows(s.history())
    ops = schedule(SEED, 4, 0, 3 * MS, 0, 40 * MS + 500_000)
    assert rows == expected_records(SEED, ops, 0)
    last = {}
    for r in rows:
        last[r[6]] = r
    assert all(r[4] == STOP for r in last.values())
    assert any(r[0] == 41 * MS for r in rows)                       # final stops at the first round past the limit
    assert max(r[0] for r in rows) == 41 * MS
    s.close()


def test_step_applies_the_nemesis_and_streamed_runs_drain_between_stretches():
    import maelstrom_b200 as mb
    rows, streamed = [], []
    for mode in ("step", "run", "streamed"):
        s = mb.Sim(10, workload="lin-kv", raft_group=5, max_endpoints=16, journal_level=1, journal_cap_log2=16)
        s.nemesis(time_limit_ns=50 * MS, interval_ns=4 * MS, start_ns=MS)
        got = []
        if mode == "step":
            for _ in range(6):
                s.step(11)
                got.append(s.history())
        elif mode == "run":
            s.run(70 * MS)
            got.append(s.history())
        else:
            for until in (13 * MS, 37 * MS + 5, 70 * MS):
                s.run_streamed(until, sink=lambda info, r, ev: streamed.append(len(ev)), fmt=8)
                got.append(s.history())
        h = nemesis_rows(np.concatenate(got))
        rows.append([r for r in h if r[0] < 66 * MS])
        s.close()
    assert rows[0] == rows[1] == rows[2] and len(rows[0]) > 10
    assert rows[1] == expected_records(SEED, schedule(SEED, 2, 0, 4 * MS, MS, 50 * MS), 0)


def test_refusals(engine_backend):
    import maelstrom_b200 as mb

    def refused(s, **kw):
        with pytest.raises(mb.SimError) as e:
            s.nemesis(**dict(dict(time_limit_ns=100 * MS), **kw))
        assert e.value.code == -2

    with mb.Sim(10, workload="lin-kv", raft_group=5, max_endpoints=16) as s:
        refused(s, group=2)                                             # not the Raft clusters
        refused(s, targets=8)
        refused(s, interval_ns=-1)
        refused(s, interval_ns=1 << 51)
        s.run(5 * MS)
        refused(s, start_ns=4 * MS)                                     # in the past
        s.partition([0] * 5 + [1] * 5)
        refused(s)                                                      # a bulk partition is installed
        s.heal()
        assert s.nemesis(time_limit_ns=100 * MS, group=5) == 0            # start_ns: now
        refused(s)                                                      # once per simulation
        with pytest.raises(mb.SimError):
            s.partition([0] * 10)                                       # the nemesis owns the component vector
        s.drop(0, 1)
        s.slow()
        s.fast()
        s.flaky()
        s.set_loss(0.0)
        s.heal()
    with mb.Sim(9, workload="broadcast", max_endpoints=16) as s:
        refused(s, group=3)                                             # gossip crosses any smaller group
    with mb.Sim(8200, workload="broadcast", n_values=64, max_endpoints=8200, ring_cap=16, max_window=16) as s:
        refused(s)                                                      # more than 8192 servers in a cluster
    with mb.Sim(10, workload="echo", max_endpoints=16, use_graph=1) as s:
        refused(s)
    if engine_backend == "emul":
        with mb.Sim(10, workload="lin-kv", raft_group=5, max_endpoints=16, n_shards=2, shard_id=0) as s:
            refused(s)


def test_clients_added_after_the_nemesis_keep_its_records():
    import maelstrom_b200 as mb
    s = mb.Sim(10, workload="lin-kv", raft_group=5, max_endpoints=64, journal_level=0)
    s.nemesis(time_limit_ns=100 * MS, interval_ns=2 * MS, start_ns=0)
    s.run(30 * MS)
    s.add_kv_clients(20, interval_ns=5 * MS, time_limit_ns=80 * MS, key_period_ns=10 * MS)   # a bigger ring
    s.run(120 * MS)
    h = s.history()
    assert nemesis_rows(h) == expected_records(SEED, schedule(SEED, 2, 0, 2 * MS, 0, 100 * MS), 0)
    assert np.count_nonzero(h["client"] != NEVER) > 0
    s.close()


def test_history_ring_overflow_names_the_nemesis():
    import maelstrom_b200 as mb
    with mb.Sim(1000, workload="lin-kv", raft_group=1, max_endpoints=1004, journal_level=0) as s:
        s.nemesis(time_limit_ns=10_000 * MS, interval_ns=1)            # ~1.5 ops per cluster and tick, never drained
        with pytest.raises(mb.SimError) as e:
            s.run(200 * MS)
        assert "history ring" in str(e.value) and "nemesis" in str(e.value)


def test_kv_history_leaves_nemesis_records_out():
    import maelstrom_b200 as mb
    rec = np.zeros(3, dtype=mb._lib.HIST_DTYPE)
    rec["client"] = [10, NEVER, 10]
    rec["f"] = [2, ONE, 2]
    rec["type"] = [0, 3, 1]
    rec["value"] = [3, 0, 3 | 4 << 16]
    assert list(mb.kv_history(rec, 10, 10)) == [(0, 3)] and len(mb.kv_history(rec, 10, 10)[(0, 3)]) == 2


# ----------------------------------------------------------------------------------------------- 6. scale (GPU)
# 819 five-node Raft clusters, 8190 kv clients.  Two seconds of nemesis interval over four seconds: about one
# partition cycle per cluster.  (Longer runs of this shape stop advancing virtual time a few cycles in: some leader
# reaches the runaway replication regime of DESIGN.md 2.3, as the host-driven nemesis of test_kv_clients.py's scale
# case does from its second cycle on.)
SCALE = dict(workload="lin-kv", latency_dist="constant", latency_mean_ms=0, server_ring_cap=64, server_max_window=32,
             rpc_table=64, n_keys=16, raft_log_cap=512, journal_cap_log2=24, ring_cap=64, max_window=32, raft_group=5)
T0 = 4500 * MS
SCALE_NEM = dict(time_limit_ns=T0 + 4000 * MS, interval_ns=2000 * MS, start_ns=T0)
STRETCHES = (1000, 2000, 3000, 4000, 4500)                          # the last one holds the final stops


def scale_scenario(n, n_clients, hist, streamed=False):
    def scenario(s, make):
        c = s.add_endpoint("c9999", O.KIND_SIM_CLIENT)
        s.schedule(ops_array([(i // 32 * MS, c, i, "init", 1 + i, 0) for i in range(n)]))
        s.run(T0)
        s.add_kv_clients(n_clients, interval_ns=1000 * MS, time_limit_ns=T0 + 2800 * MS, key_period_ns=500 * MS,
                         keys_per_group=8)
        R = make(s)
        for t in STRETCHES:
            R.run(T0 + t * MS)
            hist.append(s.history())
        return [s.raft_state(i) for i in range(0, n, 97)]
    return scenario


class Streamed:
    """R.run through ms_run_streamed (format 8), the journal collected from the batches"""

    def __init__(self, inner, batches):
        self.inner, self.batches = inner, batches

    def run(self, until):
        s = self.inner.s
        s.run_streamed(until, sink=lambda info, r, ev: self.batches.append(ev.tobytes()), fmt=8)


@pytest.mark.gpu
def test_scale_819_clusters_equal_to_the_host_driven_twin(engine_backend):
    if engine_backend != "cuda":
        pytest.skip("4095 nodes: GPU only")
    from test_kv_clients import linearizable
    import maelstrom_b200 as mb
    n, n_clients = 4095, 8190
    kw = dict(SCALE, max_endpoints=n + n_clients + 4)
    ops = schedule(SEED, n // 5, 0, SCALE_NEM["interval_ns"], T0, SCALE_NEM["time_limit_ns"])
    ha, hb = [], []
    a = mb.Sim(n, **kw)
    ra = scale_scenario(n, n_clients, ha)(a, lambda s: DeviceNemesis(s, **SCALE_NEM))
    b = mb.Sim(n, **kw)
    rb = scale_scenario(n, n_clients, hb)(b, lambda s: HostNemesis(s, SEED, n, 5, ops, T0))
    assert ra == rb
    ha, hb = np.concatenate(ha), np.concatenate(hb)
    rows = nemesis_rows(ha)
    assert rows == expected_records(SEED, ops, T0)
    assert len({r[6] for r in rows}) == n // 5                      # every cluster has its own records
    ca = ha[ha["client"] != NEVER]
    assert len(ca) == len(hb) > 4 * n
    for f in HIST_FIELDS:
        assert np.array_equal(ca[f], hb[f]), f
    ea, ba = a.drain()
    eb, bb = b.drain()
    assert len(ea) > 0 and ea.tobytes() == eb.tobytes() and ba.tobytes() == bb.tobytes()
    assert a.stats() == b.stats() and (a.now, a.round) == (b.now, b.round)
    assert a.counters()["partition_drops"] > 0
    per_key = mb.kv_history(ca[ca["client"] < n + 1 + 10 * 40], *a.kv_groups)   # the first 40 clusters
    assert len(per_key) > 40
    for key, ops_k in per_key.items():
        assert linearizable(ops_k), key
    a.close()
    b.close()


@pytest.mark.gpu
def test_scale_streamed_with_the_history_drained_between_stretches(engine_backend):
    if engine_backend != "cuda":
        pytest.skip("4095 nodes: GPU only")
    import maelstrom_b200 as mb
    n, n_clients = 4095, 8190
    kw = dict(SCALE, max_endpoints=n + n_clients + 4, journal_level=1)
    ops = schedule(SEED, n // 5, 0, SCALE_NEM["interval_ns"], T0, SCALE_NEM["time_limit_ns"])
    res = []
    for streamed in (False, True):
        s = mb.Sim(n, **kw)
        s.idle_jump()
        hist, batches = [], []
        if streamed:
            make = lambda sim: Streamed(DeviceNemesis(sim, **SCALE_NEM), batches)
        else:
            make = lambda sim: DeviceNemesis(sim, **SCALE_NEM)
        r = scale_scenario(n, n_clients, hist)(s, make)
        h = np.concatenate(hist)
        res.append((r, nemesis_rows(h), h[h["client"] != NEVER].tobytes(), s.now, s.round, s.stats(),
                    s.journal_written()))
        if streamed:
            assert len(batches) > 4 and sum(len(x) for x in batches) > 0
        s.close()
    assert res[0] == res[1]
    assert res[1][1] == expected_records(SEED, ops, T0)

