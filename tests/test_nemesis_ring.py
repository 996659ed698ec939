"""The majorities-ring target of the device partition nemesis (ms_set_nemesis targets bit 4, DESIGN.md 2.13): every
server of a partitioned cluster hears a majority of it, no two the same one, installed by k_nemesis in the cluster's
block of the pairwise [dest][src] drop matrix.  The four-target schedule and the ring are restated here from the spec,
and each run is compared with its host-driven twin: the same simulation without the nemesis, stopped at every
restated instant to install the composed component vector with ms_net_partition and each ring grudge as drop! calls
-- on the engine and, where it has the node program, on the oracle.  Journal, bodies, statistics, node and Raft
states, ms_now / ms_round and the client history must be identical; the nemesis's records must be the restated ops.
[emul] = the kernel sources on the CPU SIMT emulator, [cuda] = an H100."""
import numpy as np
import pytest

import kv_oracle_lib as K
import oracle_lib as O
from scenarios import ops_array
from test_nemesis import draw, ceil_tick, applied, nemesis_rows, outputs, assert_same

pytestmark = pytest.mark.usefixtures("engine_backend")
MS = 1_000_000
NEVER = 0xFFFFFFFF
DRAW, RANK = 0x4E454D00, 0x4E454D01
ONE, MAJORITY, MINORITY_THIRD, STOP, RING = 5, 6, 7, 8, 9
TARGET_BITS = ((1, ONE), (2, MAJORITY), (4, MINORITY_THIRD), (16, RING))   # the fixed order of a start's choice
ALL4 = 0x17
HIST_FIELDS = ("time_ns", "order", "client", "op", "type", "f", "error", "value")
SEED = 0x4D41454C


# ----------------------------------------------------------------------------------------------- the spec, restated
def schedule(seed, n_clusters, mask, interval, start, limit):
    """every op as (t_j, cluster, j, f) over the four targets: gen/stagger of the interval over a flip-flop of start /
    stop, cut at the time limit, with a final stop at the limit for a cluster left partitioned"""
    enabled = [f for bit, f in TARGET_BITS if (mask or 7) & bit]
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


def positions(seed, c, g, j):
    """ring position of each server c*g + i: its rank by (key, server)"""
    keys = sorted((draw(seed, j, c * g + i, RANK)[0], i) for i in range(g))
    out = [0] * g
    for r, (_, i) in enumerate(keys):
        out[i] = r
    return out


def sides(seed, c, g, j, f):
    m = {ONE: 1, MAJORITY: g // 2 + 1, MINORITY_THIRD: max(1, g // 3)}[f]
    return [0 if p < m else 1 for p in positions(seed, c, g, j)]


def hears(p, q, g):
    """the server at ring position p receives from the one at position q"""
    m = g // 2 + 1
    return (q - p + m // 2) % g < m


def hears_matrix(pos, g):
    """[dest member][src member] of a cluster whose member i sits at ring position pos[i]"""
    pos = np.asarray(pos, dtype=np.int64)
    m = g // 2 + 1
    return ((pos[None, :] - pos[:, None] + m // 2) % g) < m


def cut_pairs(seed, c, g, j):
    """the (src, dest) server pairs a ring start cuts"""
    h = hears_matrix(positions(seed, c, g, j), g)
    dest, src = np.nonzero(~h)
    return [(c * g + int(s), c * g + int(d)) for s, d in zip(src, dest)]


def expected_records(ops, now0):
    return [(t, NEVER, j, 3, f, 0, c) for t, group in applied(ops, now0).items() for c, j, f in group]


class HostRing:
    """the nemesis driven from the host: run() stops at every instant of the restated schedule, installs the composed
    component vector with partition() and a ring start's cut pairs with drop(); only an instant with a ring stop heals
    and re-installs everything still held.  heal() forgets every grudge, as ms_net_heal does with the nemesis on"""

    def __init__(self, sim, seed, n, g, ops, now0):
        self.s, self.seed, self.g = sim, seed, g
        self.vec = np.full(n, NEVER, dtype=np.uint32)
        self.ring = {}                                 # cluster -> its cut pairs
        self.todo = list(applied(ops, now0).items())

    def drops(self, pairs):
        for src, dest in pairs:
            self.s.drop(src, dest)

    def run(self, until):
        while self.todo and self.todo[0][0] < until:
            t, group = self.todo.pop(0)
            self.s.run(t)
            reinstall, new = False, []
            for c, j, f in group:
                lo = c * self.g
                if f == STOP and c in self.ring:
                    del self.ring[c]
                    reinstall = True
                elif f == STOP:
                    self.vec[lo:lo + self.g] = NEVER
                elif f == RING:
                    self.ring[c] = cut_pairs(self.seed, c, self.g, j)
                    new.append(c)
                else:
                    self.vec[lo:lo + self.g] = 2 * c + np.array(sides(self.seed, c, self.g, j, f), dtype=np.uint32)
            if reinstall:
                self.s.heal()
                new = list(self.ring)
            self.s.partition(self.vec)
            for c in new:
                if c in self.ring:
                    self.drops(self.ring[c])
        self.s.run(until)

    def heal(self):
        self.s.heal()
        self.vec[:] = NEVER
        self.ring = {}


class DeviceRing:
    def __init__(self, sim, **cfg):
        self.s = sim
        sim.nemesis(**cfg)

    def run(self, until):
        self.s.run(until)

    def heal(self):
        self.s.heal()


def twins(n, g, scenario, nem, oracle=None, jump=False, seed=SEED, **kw):
    """run A (device nemesis), run B (host-driven twin on the engine) and, if given, the oracle's host-driven run.
    scenario(sim, R) drives a simulation through R.run / R.heal and returns what it wants compared.
    Returns (A's outputs, A's nemesis rows, the restated ops)"""
    import maelstrom_b200 as mb
    workload = kw.get("workload", "broadcast")
    kw["seed"] = seed
    cfg = dict(nem)
    ops = schedule(seed, n // g, cfg.get("targets", 0), cfg.get("interval_ns", 0) or 10_000 * MS,
                   cfg.get("start_ns", 0), cfg["time_limit_ns"])
    a = mb.Sim(n, **kw)
    if jump:
        a.idle_jump()
    ra = scenario(a, lambda s: DeviceRing(s, **cfg))
    ha = a.history()
    oa = outputs(a, n, workload, ha)
    oa["executed"] = a.counters()["rounds"]
    oa["partition_drops"] = a.counters()["partition_drops"]
    a.close()
    rows = nemesis_rows(ha)
    assert rows == expected_records(ops, 0)
    client_a = ha[ha["client"] != NEVER]
    b = mb.Sim(n, **kw)
    rb = scenario(b, lambda s: HostRing(s, seed, n, g, ops, 0))
    ob = outputs(b, n, workload, b.history())
    b.close()
    assert ra == rb
    assert_same(dict(oa, hist=client_a), ob, "device nemesis vs host-driven twin")
    if oracle is not None:
        o = oracle()
        ro = scenario(o, lambda s: HostRing(s, seed, n, g, ops, 0))
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


# ----------------------------------------------------------------------------------------------- 1. the restatement
@pytest.mark.parametrize("seed,g,mask", [(SEED, 1, 0x10), (7, 2, 0x11), (11, 3, 0x17), (12, 4, 0x10), (13, 5, 0x17),
                                         (99, 5, 0x11), (14, 6, 0x10), (15, 7, 0x17), (5, 64, 0x10), (6, 64, 0x17)])
def test_schedule_and_ring_positions_match_the_restatement(seed, g, mask):
    import maelstrom_b200 as mb
    n = 3 * g if g < 64 else 64
    kw = dict(workload="lin-kv", raft_group=g if g < n else 0, max_endpoints=n + 4, journal_level=0, seed=seed)
    s = mb.Sim(n, **kw)
    c = s.add_endpoint("c0", O.KIND_SIM_CLIENT)
    # interval 1 ns: half of the delays are zero ticks, so several ops of a cluster share a round
    limit = 60 * MS + 300_000
    s.nemesis(time_limit_ns=limit, interval_ns=1, start_ns=2 * MS + 1, targets=mask)
    s.schedule(ops_array([(0, c, i, "init", 1 + i, 0) for i in range(n)]))
    seen = []
    s.run(30 * MS)
    seen.append(s.history())
    s.run(90 * MS)
    seen.append(s.history())
    h = np.concatenate(seen)
    ops = schedule(seed, n // g, mask, 1, 2 * MS + 1, limit)
    assert nemesis_rows(h) == expected_records(ops, 0)
    fs = {f for _, _, _, f in ops if f != STOP}
    assert fs == {f for bit, f in TARGET_BITS if mask & bit}
    rings = [(cc, j) for _, cc, j, f in ops if f == RING]
    assert rings
    for cc, j in rings[:12]:
        assert mb.nemesis_grudge(seed, cc, g, j, RING).tolist() == positions(seed, cc, g, j)
    for t, cc, j, f in ops[:24]:
        if f not in (STOP, RING):
            assert mb.nemesis_grudge(seed, cc, g, j, f).tolist() == sides(seed, cc, g, j, f)
    s.close()


@pytest.mark.parametrize("g", [1, 2, 3, 4, 5, 6, 7, 10, 64, 600, 8192])
def test_ring_properties(g):
    import maelstrom_b200 as mb
    pos = mb.nemesis_grudge(SEED, 3, g, 4, RING).astype(np.int64)
    assert sorted(pos.tolist()) == list(range(g))
    if g <= 600:
        assert pos.tolist() == positions(SEED, 3, g, 4)
    if g <= 64:
        assert all(hears(p, q, g) == bool(hears_matrix([p, q], g)[0, 1]) for p in range(g) for q in range(g))
    m = g // 2 + 1
    rows, one_way = [], False
    for lo in range(0, g, 512):                         # [dest][src] by member, 512 rows at a time
        sel = np.arange(lo, min(g, lo + 512))
        h = ((pos[None, :] - pos[sel, None] + m // 2) % g) < m
        back = ((pos[sel][None, :] - pos[:, None] + m // 2) % g).T < m   # h's transpose: does src hear dest
        assert np.all(h.sum(axis=1) == m)               # every member hears m members
        assert np.all(h[np.arange(len(sel)), sel])      # itself included
        if g <= 2:
            assert h.all()                              # nothing is cut
        one_way |= bool(np.any(h & ~back))
        rows.append(np.packbits(h, axis=1))
    if g >= 3:
        assert len(np.unique(np.concatenate(rows), axis=0)) == g   # no two members hear the same set
    assert one_way == (g >= 3 and m % 2 == 0)           # cuts are one-way exactly when m is even


def test_grudge_refusals():
    import maelstrom_b200 as mb
    with pytest.raises(mb.SimError):
        mb.nemesis_grudge(SEED, 0, 5, 0, STOP)
    with pytest.raises(mb.SimError):
        mb.nemesis_grudge(SEED, 0, 5, 0, 10)
    with pytest.raises(mb.SimError):
        mb.nemesis_grudge(SEED, 0, 8193, 0, RING)


# ----------------------------------------------------------------------------------------------- 2. twins
RAFT = dict(workload="lin-kv", latency_dist="exponential", latency_mean_ms=2, p_loss=0.02, ring_cap=256,
            max_window=128, server_ring_cap=256, server_max_window=128, rpc_table=256, n_keys=64,
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


def raft_oracle(n, g, **kw):
    return lambda: K.Sim(n, workload=O.W_RAFT, latency_dist=kw["latency_dist"], latency_mean_ms=kw["latency_mean_ms"],
                         p_loss=kw.get("p_loss", 0.0), raft_group=g, rpc_table=256, seed=kw.get("seed", SEED))


@pytest.mark.parametrize("jump", [False, True])
def test_five_node_raft_clusters_with_kv_clients_all_four_targets(jump):
    n, n_clients = 50, 100
    until = 12_000 * MS
    nem = dict(time_limit_ns=10_000 * MS, interval_ns=700 * MS, start_ns=3200 * MS, targets=ALL4)
    kw = dict(RAFT, raft_group=5, max_endpoints=n + n_clients + 4)
    oa, rows, ops = twins(n, 5, raft_scenario(n, n_clients, until), nem, oracle=raft_oracle(n, 5, **kw), jump=jump,
                          **kw)
    assert len({r[6] for r in rows}) == n // 5
    assert {r[4] for r in rows} == {ONE, MAJORITY, MINORITY_THIRD, RING, STOP}
    assert oa["stats"]["servers"]["recv-count"] > 0 and oa["partition_drops"] > 0
    if jump:
        assert oa["executed"] < 0.9 * oa["round"]


def test_six_node_raft_clusters_one_way_cuts():
    # g = 6: m = 4 is even, so a ring cuts one direction of some pairs and leaves the other
    n, n_clients = 36, 72
    until = 10_000 * MS
    nem = dict(time_limit_ns=8500 * MS, interval_ns=600 * MS, start_ns=3100 * MS, targets=0x10)
    kw = dict(RAFT, raft_group=6, max_endpoints=n + n_clients + 4)
    oa, rows, ops = twins(n, 6, raft_scenario(n, n_clients, until), nem, oracle=raft_oracle(n, 6, **kw), **kw)
    starts = [(c, j) for _, c, j, f in ops if f == RING]
    assert len(starts) > 6
    c, j = starts[0]
    cut = set(cut_pairs(SEED, c, 6, j))
    assert any((d, s) not in cut for s, d in cut)
    assert oa["partition_drops"] > 0


def test_heal_during_a_ring_partition_then_a_later_ring_cuts_again():
    n, n_clients = 20, 40
    until = 9000 * MS
    nem = dict(time_limit_ns=8000 * MS, interval_ns=900 * MS, start_ns=3000 * MS, targets=0x10)
    ops = schedule(SEED, n // 5, 0x10, 900 * MS, 3000 * MS, 8000 * MS)
    # the heal falls inside a cluster's ring partition that a later ring start of the same cluster follows
    held = [(t0, t1) for (t0, c0, j0, f0) in ops for (t1, c1, j1, f1) in ops
            if f0 == RING and c1 == c0 and j1 == j0 + 1 and ceil_tick(t1) - ceil_tick(t0) > 2 * MS
            and any(cc == c0 and f == RING and tt > t1 for tt, cc, jj, f in ops)]
    assert held
    t0, t1 = held[0]
    heal_at = ceil_tick(t0) + (ceil_tick(t1) - ceil_tick(t0)) // 2 + 1
    kw = dict(RAFT, raft_group=5, max_endpoints=n + n_clients + 4)
    oa, rows, _ = twins(n, 5, raft_scenario(n, n_clients, until, heal_at=heal_at), nem,
                        oracle=raft_oracle(n, 5, **kw), **kw)
    assert any(r[4] == RING and r[0] > heal_at for r in rows)


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


def test_broadcast_grid_with_gen_clients_ring_only():
    n = 16
    kw = dict(workload="broadcast", topology="grid", n_values=1 << 10, latency_dist="exponential", latency_mean_ms=30,
              p_loss=0.02, max_endpoints=32, ring_cap=256, max_window=128, calendar_slots=256, calendar_cap=4096)
    nem = dict(time_limit_ns=3500 * MS, interval_ns=300 * MS, start_ns=100 * MS, targets=0x10)
    oracle = lambda: O.Sim(n, workload=O.W_BROADCAST, topology="grid", n_values=1 << 10, latency_dist="exponential",
                           latency_mean_ms=30, p_loss=0.02, seed=SEED)
    oa, rows, _ = twins(n, n, broadcast_scenario, nem, oracle=oracle, **kw)
    assert len(rows) > 6 and {r[4] for r in rows} == {RING, STOP}
    assert oa["stats"]["servers"]["send-count"] > 0 and oa["partition_drops"] > 0


def gset_scenario(s, make):
    c = s.add_endpoint("c0", O.KIND_SIM_CLIENT)
    s.schedule(ops_array([(0, c, i, "init", i + 1, 0) for i in range(6)] +
                         [(t * MS, c, t % 6, "add", 100 + t, t % 50) for t in range(5, 9000, 37)]))
    R = make(s)
    R.run(12_000 * MS)
    return [s.node_set(k).tolist() for k in range(6)]


def test_gset():
    kw = dict(workload="g-set", latency_dist="constant", latency_mean_ms=20, n_values=64, max_endpoints=8,
              ring_cap=256, max_window=128, calendar_slots=64, calendar_cap=1024, gset_interval_ms=700)
    nem = dict(time_limit_ns=10_000 * MS, interval_ns=1000 * MS, start_ns=0, targets=0x12)
    oracle = lambda: O.Sim(6, workload=O.W_GSET, latency_dist="constant", latency_mean_ms=20, n_values=64,
                           gset_interval_ms=700, seed=SEED)
    oa, rows, _ = twins(6, 6, gset_scenario, nem, oracle=oracle, **kw)
    assert oa["stats"]["servers"]["send-count"] > 0 and any(r[4] == RING for r in rows)


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
    nem = dict(time_limit_ns=6000 * MS, interval_ns=400 * MS, start_ns=50 * MS, targets=ALL4)
    oracle = lambda: O.Sim(3, workload=O.W_TXN, latency_dist="constant", latency_mean_ms=5, seed=SEED)
    oa, rows, _ = twins(3, 3, txn_scenario, nem, oracle=oracle, **kw)
    assert oa["stats"]["servers"]["recv-count"] > 0 and any(r[4] == RING for r in rows)


def many_clusters_scenario(n):
    def scenario(s, make):
        c = s.add_endpoint("c0", O.KIND_SIM_CLIENT)
        s.schedule(ops_array([(i // 64 * MS, c, i, "init", 1 + i, 0) for i in range(n)]))
        R = make(s)
        R.run(1600 * MS)                              # jumped: nothing acts before the first election timeouts
        R.run(2120 * MS)                              # ops in every tick while the first elections run
        return [s.raft_state(i)["term"] for i in range(n)]
    return scenario


def test_520_three_node_clusters_share_matrix_words():
    # 520 clusters of 3: more clusters than k_nemesis has threads, and cluster blocks of 3 columns that straddle 32-bit
    # words of the pair matrix while their neighbours are healthy, in a component partition or in a ring of their own
    n = 1560
    kw = dict(workload="lin-kv", raft_group=3, max_endpoints=n + 4, ring_cap=64, max_window=64, server_ring_cap=64,
              server_max_window=64, rpc_table=64, n_keys=8, raft_log_cap=256, journal_cap_log2=22)
    nem = dict(time_limit_ns=2100 * MS, interval_ns=60 * MS, start_ns=1950 * MS, targets=ALL4)
    oa, rows, ops = twins(n, 3, many_clusters_scenario(n), nem, jump=True, **kw)
    assert len({r[6] for r in rows}) > 480 and max(r[6] for r in rows) >= 512
    assert {r[4] for r in rows} == {ONE, MAJORITY, MINORITY_THIRD, RING, STOP}
    # some round starts a ring in a cluster whose block shares a word with a neighbour's
    straddle = [c for _, c, _, f in ops if f == RING and (3 * c) // 32 != (3 * c + 2) // 32]
    assert straddle
    assert oa["stats"]["servers"]["send-count"] > 0 and oa["partition_drops"] > 0
    assert oa["executed"] < 0.5 * oa["round"]


def test_broadcast_cluster_of_600_ring_only():
    # one cluster of 600 servers: k_nemesis's rank and matrix loops stride past 512 threads, 19 words per row
    n = 600
    kw = dict(workload="broadcast", topology="grid", n_values=64, max_endpoints=n + 4, ring_cap=64, max_window=64)

    def scenario(s, make):
        c = s.add_endpoint("c0", O.KIND_SIM_CLIENT)
        s.schedule(ops_array([(t * MS, c, (t * 97) % n, "broadcast", t + 1, t % 64) for t in range(0, 40, 3)]))
        R = make(s)
        R.run(45 * MS)
        return [len(s.node_set(k)) for k in range(0, n, 37)]
    nem = dict(time_limit_ns=40 * MS, interval_ns=6 * MS, start_ns=0, targets=0x10)
    oa, rows, ops = twins(n, n, scenario, nem, **kw)
    assert sum(1 for r in rows if r[4] == RING) >= 2
    assert oa["partition_drops"] > 0
    import maelstrom_b200 as mb
    assert mb.nemesis_grudge(SEED, 0, n, rows[0][2], RING).tolist() == positions(SEED, 0, n, rows[0][2])


def test_step_applies_the_ring_and_streamed_runs_drain_between_stretches():
    import maelstrom_b200 as mb
    rows, outs = [], []
    for mode in ("step", "run", "streamed"):
        s = mb.Sim(10, workload="lin-kv", raft_group=5, max_endpoints=16, journal_level=1, journal_cap_log2=16)
        c = s.add_endpoint("c0", O.KIND_SIM_CLIENT)
        s.schedule(ops_array([(0, c, i, "init", 1 + i, 0) for i in range(10)]))
        s.nemesis(time_limit_ns=50 * MS, interval_ns=4 * MS, start_ns=MS, targets=ALL4)
        got, evs = [], []
        if mode == "step":
            for _ in range(6):
                s.step(11)
                got.append(s.history())
        elif mode == "run":
            s.run(70 * MS)
            got.append(s.history())
        else:
            for until in (13 * MS, 37 * MS + 5, 70 * MS):
                s.run_streamed(until, sink=lambda info, r, ev: evs.append(len(ev)), fmt=8)
                got.append(s.history())
            assert sum(evs) > 0
        h = nemesis_rows(np.concatenate(got))
        rows.append([r for r in h if r[0] < 66 * MS])
        if mode != "step":
            outs.append((s.now, s.round, s.stats(), [s.raft_state(i) for i in range(10)]))
        s.close()
    assert rows[0] == rows[1] == rows[2] and any(r[4] == RING for r in rows[0])
    assert rows[1] == expected_records(schedule(SEED, 2, ALL4, 4 * MS, MS, 50 * MS), 0)
    assert outs[0] == outs[1]


# ----------------------------------------------------------------------------------------------- 3. refusals, bounds
def test_refusals_and_the_pair_matrix_bound(engine_backend):
    import maelstrom_b200 as mb

    def refused(s, code=-2, **kw):
        with pytest.raises(mb.SimError) as e:
            s.nemesis(**dict(dict(time_limit_ns=100 * MS), **kw))
        assert e.value.code == code
        return str(e.value)

    with mb.Sim(10, workload="lin-kv", raft_group=5, max_endpoints=16) as s:
        assert "primaries" in refused(s, targets=8)
        refused(s, targets=0x18)
        refused(s, targets=0x20)
        refused(s, targets=0x30)
        s.drop(0, 1)
        refused(s, targets=0x10)                                        # drop! entries are installed
        s.heal()
        assert s.nemesis(time_limit_ns=100 * MS, targets=0x11) == 0
        with pytest.raises(mb.SimError) as e:
            s.drop(0, 1)                                                # the ring owns the pair matrix
        assert e.value.code == -2
        with pytest.raises(mb.SimError):
            s.partition([0] * 10)
        s.heal()
        with pytest.raises(mb.SimError):
            s.drop(2, 3)                                                # still, after a heal
        s.slow()
        s.fast()
        s.set_loss(0.0)
        s.run(120 * MS)
    with mb.Sim(10, workload="lin-kv", raft_group=5, max_endpoints=65537, ring_cap=16, max_window=16,
                server_ring_cap=16, server_max_window=16) as s:
        assert "65536" in refused(s, code=-5, targets=0x10)
        assert s.nemesis(time_limit_ns=100 * MS, targets=7) == 0       # the component targets need no matrix
    with mb.Sim(10, workload="lin-kv", raft_group=5, max_endpoints=16) as s:
        s.nemesis(time_limit_ns=100 * MS, targets=7)
        s.drop(0, 1)                                                    # without the ring drop! keeps working
        s.heal()


# ----------------------------------------------------------------------------------------------- 4. scale (GPU)
# 819 five-node Raft clusters, 8190 kv clients, the shape of test_nemesis.py's scale case but at a constant latency of
# 1 ms: at latency 0 and with the ring among the targets, virtual time stops advancing 1.905 s after the nemesis starts
# (rounds keep executing at one instant: the zero-latency loop of DESIGN.md 2.3 and 6.2, reached earlier than under
# the component targets alone)
SCALE = dict(workload="lin-kv", latency_dist="constant", latency_mean_ms=1, server_ring_cap=64, server_max_window=32,
             rpc_table=64, n_keys=16, raft_log_cap=512, journal_cap_log2=24, ring_cap=64, max_window=32, raft_group=5)
T0 = 4500 * MS
SCALE_NEM = dict(time_limit_ns=T0 + 4000 * MS, interval_ns=2000 * MS, start_ns=T0, targets=ALL4)
STRETCHES = (1000, 2000, 3000, 4000, 4500)                          # the last one holds the final stops


def scale_scenario(n, n_clients, hist):
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


@pytest.mark.gpu
def test_scale_819_clusters_all_four_targets_equal_to_the_host_driven_twin(engine_backend):
    if engine_backend != "cuda":
        pytest.skip("4095 nodes: GPU only")
    from test_kv_clients import linearizable
    import maelstrom_b200 as mb
    n, n_clients = 4095, 8190
    kw = dict(SCALE, max_endpoints=n + n_clients + 4)
    ops = schedule(SEED, n // 5, ALL4, SCALE_NEM["interval_ns"], T0, SCALE_NEM["time_limit_ns"])
    ha, hb = [], []
    a = mb.Sim(n, **kw)
    ra = scale_scenario(n, n_clients, ha)(a, lambda s: DeviceRing(s, **SCALE_NEM))
    b = mb.Sim(n, **kw)
    rb = scale_scenario(n, n_clients, hb)(b, lambda s: HostRing(s, SEED, n, 5, ops, T0))
    assert ra == rb
    ha, hb = np.concatenate(ha), np.concatenate(hb)
    rows = nemesis_rows(ha)
    assert rows == expected_records(ops, T0)
    assert len({r[6] for r in rows}) == n // 5                      # every cluster has its own records
    assert sum(1 for r in rows if r[4] == RING) > 100
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
