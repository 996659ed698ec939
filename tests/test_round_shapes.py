"""The round kernel at every CTA width and at the 8192-message window limit, against the oracle.

ms_config.threads_per_node sets the CTA width of every size class of k_round: any multiple of 32 in [32, 512], or 0
for the classes' own widths (64 / 128 / 256 / 512; g-set 256 / 256 / 256 / 512).  Classes 0-2 are compiled for at
most 256 threads, so 480 and 512 widen class 3 only (on the H100 a wider launch of them fails).  What depends on
the width: the per-thread window segments of the block-start scan (a bit mask of block starts only while a segment
has <= 32 slots), the strided loops of the bitonic fallback, the thread that claims the journal chunk (32 % nt), the
number of warps in the block scans (1 to 16), widths that are not powers of two, and on the sending side how
emissions claim ring space: per warp, which at 32 threads is per CTA.  That last one changes the sender blocks a
receiver sees, so how many windows need the bitonic sort (counters()["fallback_sorts"]) depends on the width and is
never compared across widths.

max_window may be up to 8192.  Class 3 then takes windows of 2049 to 8192 messages (its work list split at 5120:
longer windows are filled in from the front), the 16-bit shared-memory indices (ord, tab, s_bstart, s_boff, s_S)
and the 16-bit per-neighbour counts of the packed scan reach their largest values, the service walks 8192 requests
on one thread, and a CTA takes 25 B of dynamic shared memory per slot.  Which windows a run reached is counted from
its journal, as :recv events per (destination, round): counters()["max_window"] only sees broadcast and g-set
server windows.

Every case compares with the oracle as test_counter_origins.run_case does: the level-2 journal field by field,
bodies, stats, now, round, node sets, compact-ring accounting where the scenario qualifies, closed-loop client
histories, and what the scenario returns (client replies, Raft states).  The width matrix also checks that every
width gives byte-identical outputs to the default one: widths 32, 96 and 160 on the families' small scenarios, 480 and
512 on variants with a class-3 window.  The emulator ([emul], CPU suite) runs all but the Raft and hash-tree variants
at 480 and 512; the H100 ([cuda]) runs the whole matrix."""
import contextlib

import numpy as np
import pytest

import oracle_lib as O
import test_counter_origins as T
from scenarios import make_pair, ops_array, random_broadcast_ops
from test_cta_interleave import SEEDS, ctas, overlapped   # noqa: F401 (ctas is a fixture)

pytestmark = pytest.mark.usefixtures("engine_backend")
cuda_only = pytest.mark.gpu

MS = 1_000_000
RECV = np.uint64(1 << 63)
WIDTHS = (32, 96, 160, 480, 512)


@contextlib.contextmanager
def cta_width(nt):
    """Every maelstrom_b200.Sim created inside runs k_round with nt threads per CTA (0: the classes' own widths)."""
    import maelstrom_b200 as mb
    base = mb.Sim

    class Sim(base):
        def __init__(self, *a, **kw):
            kw.setdefault("threads_per_node", nt)
            super().__init__(*a, **kw)
    mb.Sim = Sim
    try:
        yield
    finally:
        mb.Sim = base


def run(case, nt):
    with cta_width(nt):
        return T.run_case(case, None)


def windows(ev):
    """(dest, size) of every window in a journal.  Inside a round the endpoints' :recv events come in runs, one per
    endpoint, each followed by that endpoint's :send events (DESIGN.md 2.3), and delta rounds share a time: a window
    is a run of :recv events of one destination at one time.  (Two windows of an endpoint that sends nothing, in
    consecutive rounds, may read as one; every endpoint whose windows the cases below target sends.)"""
    recv = (ev["event_id"] & RECV) != 0
    dest = ev["dest"].astype(np.int64)
    cont = np.zeros(len(ev), dtype=bool)
    cont[1:] = recv[1:] & recv[:-1] & (dest[1:] == dest[:-1]) & (ev["time_ns"][1:] == ev["time_ns"][:-1])
    label = np.cumsum(~cont)
    size = np.bincount(label[recv])
    first = recv & ~cont
    return list(zip(dest[first].tolist(), size[label[first]].tolist()))


def window_sizes(ev):
    return {k for _, k in windows(ev)}


def counters_into(seen, s):
    if T.is_engine(s):
        seen.update(s.counters())


# ------------------------------------------------------------------------------------------- scenarios
def bcast_general(hot=0):
    # exponential latency and loss (Philox draws, the timing wheel, the general emission path), a partition and heal;
    # hot > 0: first a burst of that many values from a client to server 5 (a window of hot messages)
    n = 16
    sizing = (dict(n_values=4096, ring_cap=4096, max_window=4096) if hot else
              dict(n_values=1024, ring_cap=1024, max_window=512, calendar_cap=4096))

    def make():
        g, o = make_pair(n, topology="grid", latency_dist="exponential", latency_mean_ms=3, p_loss=0.05,
                         journal_cap_log2=20, max_endpoints=n + 8, calendar_slots=256, **sizing)

        def scenario(s, body):
            cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(3)]
            if hot:
                s.schedule(flood(cs[0], 5, hot, v0=1000, mid0=10000))
            ops, _ = random_broadcast_ops(n, cs, n_ticks=10, per_tick=20, seed=19)
            s.schedule(ops)
            s.run(4 * MS)
            s.partition([(i // 4) % 2 for i in range(n)])
            s.run(14 * MS)
            s.heal()
            s.run(120 * MS)
        return g, o, scenario
    return T.Case(make, True, node_sets=n)


def raft_kv_clients():
    # closed-loop lin-kv clients on the device against the kv-oracle twin; the Raft states are returned and compared
    from test_kv_clients import T0, raft_pair, start
    n, nc = 5, 10

    def make():
        g, o = raft_pair(n, nc)

        def scenario(s, body):
            start(s, n)
            c0 = s.add_kv_clients(nc, interval_ns=20 * MS, time_limit_ns=T0 + 300 * MS, key_period_ns=100 * MS,
                                  keys_per_group=4)
            s.run(T0 + 500 * MS)
            return c0, [s.raft_state(i) for i in range(n)]
        return g, o, scenario
    return T.Case(make, True, history=True)


# ------------------------------------------------------------------------------------------- window builders
BIG = dict(ring_cap=8192, max_window=8192, journal_cap_log2=21)


def flood(client, dest, k, v0=0, t_ns=0, mid0=0):
    """k broadcast ops from one client to `dest` at t_ns, values v0 .. v0 + k - 1"""
    return ops_array([(t_ns, client, dest, "broadcast", mid0 + i + 1, v0 + i) for i in range(k)])


def one_block(k, seen):
    """5-node line: k values to server 2 in one round; the round after, servers 1 and 3 each receive them as one
    sender block of k compact records from server 2."""
    def make():
        g, o = make_pair(5, topology="line", n_values=k + 8, max_endpoints=8, **BIG)

        def scenario(s, body):
            c = s.add_endpoint("c0", O.KIND_SIM_CLIENT)
            s.schedule(flood(c, 2, k))
            s.run(6 * MS)
            counters_into(seen, s)
        return g, o, scenario
    return T.Case(make, False, compact="eq", node_sets=5)


def mixed(k_g, k_f, seen):
    """5-node line: k_g values to server 2, then k_f values to server 1 the round after.  Server 1's next window is
    k_f 48-B records from the client's injector slices and k_g compact records from server 2."""
    def make():
        # rings of 16384: server 3 holds a window of the filler from server 4 while server 2 claims k_f more
        g, o = make_pair(5, topology="line", n_values=k_g + k_f + FILLER + 8, max_endpoints=8, server_max_window=8192,
                         **dict(BIG, ring_cap=16384))

        def scenario(s, body):
            c = s.add_endpoint("c0", O.KIND_SIM_CLIENT)
            inject_two_rounds(s, c, k_g, k_f)
            s.run(8 * MS)
            counters_into(seen, s)
        return g, o, scenario
    return T.Case(make, False, compact="eq", node_sets=5)


FILLER = 4096


def filler(k_f):
    return min(FILLER, 8192 - k_f)      # the client's window of broadcast_ok replies stays within 8192


def inject_two_rounds(s, c, k_g, k_f):
    """k_g values to server 2 in one round; in the next (a delta round at the same time) k_f values to server 1
    interleaved with filler(k_f) values to server 4.  The filler gives every injector slice more messages than a CTA of 512
    threads emits in one pass, so a warp claims ring space for server 1 in more than one pass: the claims of
    different warps interleave, server 1's sender blocks overlap, and its window is sorted by the bitonic fallback,
    its per-neighbour counts by the packed 16-bit scan (agg_mode 2)."""
    s.schedule(flood(c, 2, k_g))
    s.step(1)
    k = k_f + filler(k_f)
    to_one = np.zeros(k, dtype=bool)
    to_one[np.linspace(0, k - 1, k_f).astype(np.int64) if k_f else []] = True
    rows = flood(c, 4, k, v0=k_g, mid0=k_g)
    rows["dest"][to_one] = 1
    s.schedule(rows)


def txn_hammer(counts, seen, n_clients=16):
    """len(counts) single-key txn nodes, node i receiving counts[i] txns, all at once; the round after, each sends one
    read per txn to lin-kv: a service window of sum(counts) requests in (at least) one sender block per node"""
    n, k = len(counts), int(sum(counts))

    def make():
        g, o = make_pair(n, workload="txn-list-append", max_endpoints=n + n_clients + 4, **BIG)

        def scenario(s, body):
            kv = s.add_endpoint("lin-kv", O.KIND_SERVICE)
            cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(n_clients)]
            rows = np.zeros(k, dtype=O.OP_DTYPE)
            rows["src"] = np.asarray(cs, dtype=np.uint32)[np.arange(k) % n_clients]
            rows["dest"] = np.repeat(np.arange(n), counts)
            b = rows["body"]
            b["type"] = O.T["txn"]
            b["flags"] = O.F_MSG_ID | np.where(np.arange(k) % 3 == 0, O.F_APPENDS, 0)
            b["msg_id"] = 1 + np.arange(k) // n_clients
            b["p1"] = 1000 + np.arange(k)
            s.schedule(rows)
            s.run(10 * MS)
            counters_into(seen, s)
            return kv, s.client_replies()
        return g, o, scenario
    return T.Case(make, False)


def spread(n, k):
    """k txns over n nodes, as even as can be"""
    return [k // n + (i < k % n) for i in range(n)]


def service_hammer(svc, k, seen, n_clients=64, max_window=8192):
    """k requests to one service in one round, from n_clients clients (k / n_clients replies each)"""
    n = 4

    def make():
        g, o = make_pair(n, topology="grid", n_values=64, max_endpoints=n + n_clients + 4,
                         **dict(BIG, max_window=max_window))

        def scenario(s, body):
            sv = s.add_endpoint(svc, O.KIND_SERVICE)
            cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(n_clients)]
            rng = np.random.default_rng(k)
            rows = np.zeros(k, dtype=O.OP_DTYPE)
            rows["src"] = np.asarray(cs, dtype=np.uint32)[np.arange(k) % n_clients]
            rows["dest"] = sv
            b = rows["body"]
            kind = rng.integers(0, 3, size=k)
            b["type"] = np.array([O.T["read"], O.T["write"], O.T["cas"]])[kind]
            b["flags"] = O.F_MSG_ID | np.where((kind == 2) & (rng.integers(0, 2, size=k) == 1), O.F_CREATE, 0)
            b["msg_id"] = 1 + np.arange(k) // n_clients
            b["p0"] = rng.integers(0, 6, size=k)
            b["p1"] = rng.integers(0, 4, size=k) | np.where(kind == 2, rng.integers(0, 4, size=k) << 32, 0)
            s.schedule(rows)
            s.run(6 * MS)
            counters_into(seen, s)
            return sv, s.client_replies()
        return g, o, scenario
    return T.Case(make, True)


def gset_adds(k, seen):
    """3 g-set nodes; k adds to node 0 in one round (its replicate_one messages then give the others k as well)"""
    n = 3

    def make():
        g, o = make_pair(n, workload="g-set", n_values=k + 8, max_endpoints=n + 20, gset_interval_ms=5000, **BIG)

        def scenario(s, body):
            cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(16)]
            s.schedule(ops_array([(0, cs[0], i, "init", 9000 + i, 0) for i in range(n)]))
            s.schedule(ops_array([(MS, cs[i % 16], 0, "add", 1 + i // 16, i) for i in range(k)]))
            s.run(8 * MS)
            counters_into(seen, s)
            return s.client_replies()
        return g, o, scenario
    return T.Case(make, False, node_sets=n)


def wheel(k, seen):
    """5-node line, constant latency 2: k values to server 2 at once, released from the timing wheel in one tick;
    two ticks later servers 1 and 3 receive its gossip of them in one window each"""
    def make():
        g, o = make_pair(5, topology="line", latency_dist="constant", latency_mean_ms=2, n_values=k + 8,
                         max_endpoints=8, calendar_slots=64, **BIG)

        def scenario(s, body):
            c = s.add_endpoint("c0", O.KIND_SIM_CLIENT)
            s.schedule(flood(c, 2, k))
            s.run(20 * MS)
            counters_into(seen, s)
        return g, o, scenario
    return T.Case(make, False, node_sets=5)


def grid3(per_tick, seen):
    """3 x 3 grid, every value injected at the centre: each corner hears every value from both of its neighbours in
    the same round, a window of exactly 2 * per_tick in two compact blocks"""
    def make():
        g, o = make_pair(9, topology="grid", n_values=per_tick + 8, max_endpoints=12, **BIG)

        def scenario(s, body):
            c = s.add_endpoint("c0", O.KIND_SIM_CLIENT)
            s.schedule(flood(c, 4, per_tick))
            s.run(8 * MS)
            counters_into(seen, s)
        return g, o, scenario
    return T.Case(make, False, compact="eq", node_sets=9)


def burst(workload, k, n=4, n_clients=16):
    """n echo or g-set nodes; k requests to node 1 in one round, from n_clients clients: a window of k"""
    def make():
        g, o = make_pair(n, workload=workload, topology="grid", n_values=k + 8, max_endpoints=n + n_clients + 4,
                         gset_interval_ms=7, **BIG)

        def scenario(s, body):
            cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(n_clients)]
            if workload == "g-set":
                s.schedule(ops_array([(0, cs[0], i, "init", 9000 + i, 0) for i in range(n)]))
            rows = np.zeros(k, dtype=O.OP_DTYPE)
            rows["time_ns"] = MS
            rows["src"] = np.asarray(cs, dtype=np.uint32)[np.arange(k) % n_clients]
            rows["dest"] = 1
            b = rows["body"]
            b["type"] = O.T["echo" if workload == "echo" else "add"]
            b["flags"] = O.F_MSG_ID
            b["msg_id"] = 1 + np.arange(k) // n_clients
            b["p0"] = np.arange(k)
            b["p1"] = np.arange(k) * 977
            s.schedule(rows)
            s.run(30 * MS)
            return s.client_replies()
        return g, o, scenario
    return T.Case(make, False, node_sets=n if workload == "g-set" else 0)


def services_burst(k, n_clients=64):
    """k requests to each of the four services in one round"""
    n = 4

    def make():
        g, o = make_pair(n, topology="grid", n_values=64, max_endpoints=n + n_clients + 8, **BIG)

        def scenario(s, body):
            sv = [s.add_endpoint(name, O.KIND_SERVICE) for name in ("lin-kv", "seq-kv", "lww-kv", "lin-tso")]
            cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(n_clients)]
            rng = np.random.default_rng(k)
            m = 4 * k
            rows = np.zeros(m, dtype=O.OP_DTYPE)
            rows["src"] = np.asarray(cs, dtype=np.uint32)[np.arange(m) % n_clients]
            rows["dest"] = np.asarray(sv, dtype=np.uint32)[np.arange(m) % 4]
            b = rows["body"]
            kind = rng.integers(0, 3, size=m)
            b["type"] = np.where(np.arange(m) % 4 == 3, O.T["ts"], np.array([O.T["read"], O.T["write"], O.T["cas"]])[kind])
            b["flags"] = O.F_MSG_ID | np.where((kind == 2) & (rng.integers(0, 2, size=m) == 1), O.F_CREATE, 0)
            b["msg_id"] = 1 + np.arange(m) // n_clients
            b["p0"] = rng.integers(0, 6, size=m)
            b["p1"] = rng.integers(0, 4, size=m) | np.where(kind == 2, rng.integers(0, 4, size=m) << 32, 0)
            s.schedule(rows)
            s.run(6 * MS)
            return s.client_replies()
        return g, o, scenario
    return T.Case(make, True)


def raft_burst(k, n=3):
    """3 Raft nodes; once a leader is elected, k reads and writes to node 0 in one round.  (The closed-loop kv clients
    keep one request per client in flight, so their windows stay small.)"""
    def make():
        g, o = make_pair(n, workload="lin-kv", n_values=256, max_endpoints=n + 20, journal_cap_log2=21,
                         ring_cap=4096, max_window=4096, raft_log_cap=8192)

        def scenario(s, body):
            cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(16)]
            s.schedule(ops_array([(0, cs[0], i, "init", 9000 + i, 0) for i in range(n)]))
            rows = np.zeros(k, dtype=O.OP_DTYPE)
            rows["time_ns"] = 2500 * MS
            rows["src"] = np.asarray(cs, dtype=np.uint32)[np.arange(k) % 16]
            b = rows["body"]
            b["type"] = np.where(np.arange(k) % 2 == 0, O.T["read"], O.T["write"])
            b["flags"] = O.F_MSG_ID
            b["msg_id"] = 1 + np.arange(k) // 16
            b["p0"] = np.arange(k) % 4
            b["p1"] = np.arange(k) % 5
            s.schedule(rows)
            s.run(2700 * MS)
            return s.client_replies(), [s.raft_state(i) for i in range(n)]
        return g, o, scenario
    return T.Case(make, True)


def tree_burst(n):
    """n hash-tree nodes (the benchmark's table sizes), one txn each at once: lin-kv's window of n root reads.  (A
    node serves one txn at a time, so a big window at a node itself runs out of its staging capacity.)"""
    from test_txn_tree import txn_ops

    def make():
        g, o = make_pair(n, workload="txn-list-append-tree", max_endpoints=n + 24, ring_cap=4096, max_window=4096,
                         server_ring_cap=64, server_max_window=32, rpc_table=64, tree_ptrs=1024, journal_cap_log2=22,
                         seed=977)

        def scenario(s, body):
            s.add_endpoint("lin-kv", O.KIND_SERVICE)
            s.add_endpoint("lww-kv", O.KIND_SERVICE)
            cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(16)]
            s.schedule(ops_array([(0, cs[i % 16], i, "init", 1 + i // 16, 0) for i in range(n)]))
            rows = txn_ops(np.random.default_rng(3), n, cs, 5, 1, n, 8, [1000] * 16)
            rows["dest"] = np.arange(n)
            s.schedule(rows)
            s.run(300 * MS)
            return s.client_replies()
        return g, o, scenario
    return T.Case(make, True)


# ------------------------------------------------------------------------------------------- width matrix
# Widths up to 256 apply to every size class: the families' small scenarios (windows of at most 512, classes 0-1).
FAMILIES = {
    "bcast_compact": T.SCENARIOS["bcast_compact"],   # latency 0, grid: compact gossip, per-neighbour block claims
    "bcast_general": bcast_general(),
    "echo": T.SCENARIOS["echo"],
    "gset": T.SCENARIOS["gset"],
    "services": T.SCENARIOS["services"],             # lin-kv, seq-kv, lww-kv, lin-tso
    "txn": T.SCENARIOS["txn"],
    "raft_kv_clients": raft_kv_clients(),
    "txn_tree": T.SCENARIOS["txn_tree"],
}
# Wider CTAs run class 3 only (max_window 4096 or more), so at 480 and 512 threads each family runs a variant with a
# window of more than 2048 messages, and the case asserts that the journal shows one.
WIDE = 2600
WIDE_FAMILIES = {
    "bcast_compact": grid3(WIDE // 2, {}),           # corner windows of WIDE in two compact blocks
    "bcast_general": bcast_general(hot=WIDE),
    "echo": burst("echo", WIDE),
    "gset": burst("g-set", WIDE),
    "services": services_burst(WIDE),
    "txn": txn_hammer(spread(100, WIDE), {}),        # lin-kv's window of WIDE reads
    "raft": raft_burst(WIDE),
    "txn_tree": tree_burst(2100),
}
# the emulator's cases at 480 and 512 threads: all but the two slowest
EMUL_WIDE = ("bcast_compact", "bcast_general", "echo", "gset", "services", "txn")

_BASE = {}


def base_run(name, backend, wide):
    """The family's scenario at the default widths, once per backend."""
    key = (name, backend, wide)
    if key not in _BASE:
        _BASE[key] = run((WIDE_FAMILIES if wide else FAMILIES)[name], 0)
    return _BASE[key]


def matrix():
    for name in FAMILIES:
        for nt in (32, 96, 160):
            yield pytest.param(name, nt, id="%s-%d" % (name, nt))
    for name in WIDE_FAMILIES:
        for nt in (480, 512):
            yield pytest.param(name, nt, marks=[] if name in EMUL_WIDE else [cuda_only], id="%s_wide-%d" % (name, nt))


@pytest.mark.parametrize("name,nt", list(matrix()))
def test_width_matrix(engine_backend, name, nt):
    wide = nt > 256
    case = (WIDE_FAMILIES if wide else FAMILIES)[name]
    res = run(case, nt)
    if wide:
        assert max(window_sizes(res["ev"])) > 2048          # a class-3 CTA of nt threads ran
    # metamorphic: the width decides how a round is computed, never what it computes
    base = base_run(name, engine_backend, wide)
    for f in ("event_id", "time_ns", "msg_id", "src", "dest"):
        assert np.array_equal(res["ev"][f], base["ev"][f]), f
    for f in ("id", "type", "flags", "msg_id", "in_reply_to", "p0", "p1"):
        assert np.array_equal(res["bd"][f], base["bd"][f]), f
    assert (res["stats"], res["now"], res["round"], res["sets"]) == (base["stats"], base["now"], base["round"],
                                                                     base["sets"])
    assert res["ret"] == base["ret"]
    if "history" in base:
        for f in ("time_ns", "order", "client", "op", "type", "f", "error", "value"):
            assert np.array_equal(res["history"][f], base["history"][f]), f
    if case.compact == "eq":
        assert res["compact"] == base["compact"] > 0
    assert len(res["ev"]) > 300


# ------------------------------------------------------------------------------------------- segments and fallback
@pytest.mark.parametrize("nt", [32, 96, 160])
def test_segments_longer_than_32_slots(nt):
    # a window of 32 * nt + 1 slots gives every thread a segment of 33: block starts are found without the bit mask.
    # (At 256 threads and more that would take a window above 8192, and the default widths never get there.)
    k = 32 * nt + 1
    seen = {}
    res = run(one_block(k, seen), nt)
    got = windows(res["ev"])
    assert (1, k) in got and (3, k) in got          # the single-block windows of servers 1 and 3
    assert seen["max_window"] == k


@pytest.mark.parametrize("nt", (0,) + WIDTHS)
def test_bitonic_fallback_at_every_width(nt):
    # 100 txn nodes each send reads to lin-kv in the same round: 100 sender tickets, more than the 64 blocks the fast
    # ordering path takes, whatever the width.  Nodes 50-99 have windows of 70 txns, in the upper half of the smallest
    # size class, whose tickets are taken first: their reads reach lin-kv before those of nodes 0-49, out of order.
    counts = [1] * 50 + [70] * 50
    seen = {}
    res = run(txn_hammer(counts, seen), nt)
    kv, replies = res["ret"]
    assert (kv, sum(counts)) in windows(res["ev"])
    assert seen["fallback_sorts"] > 0
    assert replies == sum(counts)                   # every txn answered


# ------------------------------------------------------------------------------------------- the 8192 limit
SIZES = (4097, 5120, 5121, 8191, 8192)


@pytest.mark.parametrize("k", SIZES)
def test_single_sender_block(k):
    seen = {}
    res = run(one_block(k, seen), 0)
    got = windows(res["ev"])
    assert (1, k) in got and (3, k) in got and (2, k) in got
    assert seen["max_window"] == k


@pytest.mark.parametrize("k", SIZES)
def test_more_than_64_sender_blocks(k):
    # 128 txn nodes: lin-kv's window is sorted by the bitonic fallback, up to np = 8192
    seen = {}
    res = run(txn_hammer(spread(128, k), seen), 0)
    kv, replies = res["ret"]
    assert (kv, k) in windows(res["ev"])
    assert seen["fallback_sorts"] > 0 and replies == k


@pytest.mark.parametrize("k_g,k_f", [(4097, 4095), (5121, 3071), (8191, 1), (1, 8191)])
def test_mixed_server_window(k_g, k_f):
    # server_max_window = 8192: the 48-B and compact parts of server 1's window add up to it
    seen = {}
    res = run(mixed(k_g, k_f, seen), 0)
    got = windows(res["ev"])
    assert (1, k_g + k_f) in got and (4, filler(k_f)) in got
    assert seen["max_window"] == 8192
    if k_f + filler(k_f) > 8 * 512:
        assert seen["fallback_sorts"] > 0


@pytest.mark.parametrize("svc", ["lin-kv", "seq-kv", "lww-kv"])
def test_service_walks_8192_requests(svc):
    seen = {}
    res = run(service_hammer(svc, 8192, seen), 0)
    sv, replies = res["ret"]
    assert (sv, 8192) in windows(res["ev"])
    assert replies == 8192


def test_gset_node_takes_8192_adds():
    seen = {}
    res = run(gset_adds(8192, seen), 0)
    assert (0, 8192) in windows(res["ev"])
    assert seen["max_window"] == 8192
    assert res["ret"] == 8192 + 3                   # add_ok and init_ok replies


@pytest.mark.parametrize("k", [5121, 8192])
def test_window_released_from_the_timing_wheel(k):
    seen = {}
    res = run(wheel(k, seen), 0)
    got = windows(res["ev"])
    assert (2, k) in got and (1, k) in got and (3, k) in got
    assert seen["max_window"] == k


def test_grid_corners_hear_two_neighbours():
    seen = {}
    res = run(grid3(4096, seen), 0)
    got = windows(res["ev"])
    assert all((c, 8192) in got for c in (0, 2, 6, 8))
    assert seen["max_window"] == 8192


@pytest.mark.parametrize("where", ["server", "service"])
def test_window_of_8193_is_refused(where):
    import maelstrom_b200 as mb
    if where == "server":
        # both parts fit their rings (server_ring_cap 8192 each), their sum does not fit the window
        g = mb.Sim(5, topology="line", n_values=12300, max_endpoints=8, server_max_window=8192, **BIG)
        c = g.add_endpoint("c0", O.KIND_SIM_CLIENT)
        inject_two_rounds(g, c, 4097, 4096)
        victim = 1
    else:
        g = mb.Sim(4, topology="grid", n_values=64, max_endpoints=80, **dict(BIG, ring_cap=16384))
        victim = g.add_endpoint("lin-kv", O.KIND_SERVICE)
        cs = [g.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(64)]
        g.schedule(ops_array([(0, cs[i % 64], victim, "read", 1 + i // 64, 0) for i in range(8193)]))
    with pytest.raises(mb.SimError) as e:
        g.run(8 * MS)
    msg = str(e.value)
    assert "per-round window exceeds" in msg and ("at endpoint %d " % victim) in msg, msg
    g.close()


# ------------------------------------------------------------------------------------------- refusals
def test_sizes_out_of_range_are_refused():
    import maelstrom_b200 as mb

    def refused(**kw):
        with pytest.raises(mb.SimError) as e:
            mb.Sim(5, topology="line", **kw)
        return str(e.value)
    assert "max_window must be <= 8192" in refused(ring_cap=16384, max_window=16384)
    for nt in (16, 100, 544):
        assert "threads_per_node must be a multiple of 32" in refused(threads_per_node=nt)
    assert "server_max_window must not exceed max_window" in refused(ring_cap=4096, max_window=1024,
                                                                      server_max_window=2048)


def test_max_window_rounds_up_to_a_power_of_two():
    # max_window 5000 is 8192: a service window of 8192 requests runs
    res = run(service_hammer("lin-kv", 8192, {}, max_window=5000), 0)
    assert (res["ret"][0], 8192) in windows(res["ev"])


# ------------------------------------------------------------------------------------------- concurrency, shards
def test_concurrent_ctas_at_width_96(ctas):
    L = ctas(SEEDS[0], each=True)
    seen = {}
    res = run(txn_hammer(spread(128, 8192), seen), 96)
    assert (res["ret"][0], 8192) in windows(res["ev"]) and seen["fallback_sorts"] > 0
    overlapped(L, b"k_round")


def test_two_shards_at_width_96(engine_backend):
    if engine_backend != "emul":
        pytest.skip("emulated shards: two GPUs are tests/test_gpu_sharded.py")
    from test_emul_sharded import check_against_oracle, run_sharded_scenario
    n = 36
    kw = dict(topology="grid", n_values=2048, seed=31)

    def scenario(s, body):
        cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(3)]
        ops, _ = random_broadcast_ops(n, cs, n_ticks=6, per_tick=200, seed=37)
        s.schedule(ops)
        s.run(20 * MS)

    sim_kw = dict(workload="broadcast", ring_cap=4096, max_window=4096, journal_cap_log2=20, max_endpoints=n + 8,
                  threads_per_node=96, **kw)
    ev, st, now, rnd = run_sharded_scenario(2, n, sim_kw, scenario)
    o = O.Sim(n, workload=O.W_BROADCAST, **kw)
    check_against_oracle(o, scenario, ev, st, now, rnd)
    assert max(window_sizes(ev)) > 96                # windows that take a CTA of 96 more than one pass


# ------------------------------------------------------------------------------------------- benchmark topology
@cuda_only
@pytest.mark.parametrize("nt", [0, 96])
def test_bench_topology_windows_above_4096(nt):
    # the 64 x 64 grid of bench.py with one hot node: it takes ~2280 values in one round, and the nodes on its
    # diagonals hear each of them from two neighbours in the same round, windows of ~4560 in class 3
    from test_gpu_parity import hot_broadcast_ops
    n, V = 4096, 2400
    with cta_width(nt):
        g, o = make_pair(n, topology="grid", n_values=V + 8, max_endpoints=n + 8, ring_cap=8192, max_window=8192,
                         journal_cap_log2=27, journal_level=1)
    for s in (g, o):
        cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(4)]
        s.schedule(hot_broadcast_ops(n, cs, 1, V, [32 * 64 + 32], 950, seed=78))
        s.run(MS)
    ev_g, _ = g.drain(bodies=False)
    ev_o, _ = o.journal()
    assert len(ev_g) == len(ev_o)
    for f in ("event_id", "time_ns", "msg_id", "src", "dest"):
        assert np.array_equal(ev_g[f], ev_o[f]), f
    assert g.stats() == o.stats() and g.now == o.now and g.round == o.round
    assert [g.node_set(k).size for k in (0, n - 1)] == [V, V]
    assert 4096 < g.counters()["max_window"] == max(window_sizes(ev_o)) <= 8192
    g.close()
