"""The engine across the 32-bit boundaries of its counters.

A benchmark run hands out message ids past 2^32 and event ids past 2^33, and long runs take rounds past the 15-bit
tags of the per-ticket tables; every inbox ring counter is a u32 that wraps.  ms_set_origin (Sim.set_origin)
starts a fresh simulation as if that many rounds, messages and events had happened, with the ring counters of
endpoint e at ring_pos + e * ring_stride, and the oracle's or_set_origin does the same for its counters.  Each
case places one boundary (or all of them) in the busy middle of an existing scenario and checks:

- parity: the level-2 journal, stats, now, round and node sets equal the oracle's at the same origin, and the
  compact-ring accounting of ring_counters() holds (counters taken modulo 2^32);
- non-vacuity: the boundary really was crossed, inside a round (ids / events), with some ring counter wrapped
  while its window was still open (rings), or with the final round past the boundary (rounds);
- the metamorphic relation, which also catches a mistake the oracle shares: an origin of message id, event id or
  ring position reproduces the origin-0 journal with ids shifted by the constants, and the same stats; a round
  origin does the same for scenarios that draw nothing from Philox (whose counter is the round).

Every case runs on the emulator ([emul], CPU suite) and on the H100 ([cuda])."""
import ctypes as C
import json

import numpy as np
import pytest

import oracle_lib as O
from scenarios import both, make_pair, oracle_gossip_sends, random_broadcast_ops

pytestmark = pytest.mark.usefixtures("engine_backend")
cuda_only = pytest.mark.gpu

B32 = 1 << 32
B31 = 1 << 31
B15 = 1 << 15
EVENT_MASK = np.uint64((1 << 63) - 1)
RECV = np.uint64(1 << 63)


def is_engine(s):
    return hasattr(s, "ring_counters")


# ------------------------------------------------------------------------------------------- scenarios
# Each builder returns a Case: make() -> (engine, oracle, scenario(s, body)), and what holds for it.
class Case:
    def __init__(self, make, philox, compact=None, node_sets=0, history=False, recv=None):
        self.make = make              # () -> (g, o, scenario)
        self.philox = philox          # draws from Philox: a round origin changes its journal
        self.compact = compact        # "eq" / "le" / None: compact-ring accounting against the oracle's gossip
        self.node_sets = node_sets    # servers whose node_set is compared
        self.history = history        # closed-loop clients: ms_hist records are compared
        self.recv = recv


def bcast(n=16, topo="grid", latency=0, dist="constant", ticks=8, per_tick=20, seed=3, **sizing):
    def make():
        g, o = make_pair(n, topology=topo, latency_dist=dist, latency_mean_ms=latency, n_values=1024,
                         ring_cap=1024, max_window=512, journal_cap_log2=20, max_endpoints=n + 8, calendar_slots=256,
                         calendar_cap=4096, **sizing)

        def scenario(s, body):
            cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(3)]
            ops, _ = random_broadcast_ops(n, cs, n_ticks=ticks, per_tick=per_tick, seed=seed)
            s.schedule(ops)
            s.run((ticks + 20 + 30 * latency) * 1_000_000)
        return g, o, scenario
    philox = dist != "constant"
    return Case(make, philox, compact="eq" if latency == 0 else None, node_sets=n)


def mixed(k_g, k_f):
    from test_compact_gossip import mixed_window

    def make():
        g, o, scenario, _ = mixed_window(k_g, k_f, server_ring_cap=4096, server_max_window=2048)
        return g, o, scenario
    return Case(make, False, compact="eq", node_sets=5)


def ring_wrap(cap):
    from test_compact_gossip import both_rings_wrap

    def make():
        g, o, scenario, _ = both_rings_wrap(cap)
        return g, o, scenario
    return Case(make, False, compact="eq", node_sets=5)


def phases(change_name):
    import test_compact_gossip as T
    change = getattr(T, change_name)

    def make():
        g, o = make_pair(16, topology="grid", n_values=1024, ring_cap=1024, max_window=512, journal_cap_log2=20,
                         max_endpoints=24)
        scenario, _ = T.phase_scenario(change)
        return g, o, scenario
    philox = change_name in ("loss_on_off", "flaky")
    return Case(make, philox, compact="eq" if change_name in ("partition_heal", "drop_pair") else "le", node_sets=16)


def remove_readd():
    # a host endpoint (not a client: server replies to it take the latency) is removed while replies to it wait in
    # the timing wheel, and its slot goes to a new host endpoint: k_release must drop what was sent before the new
    # endpoint was born (ep_born, compared with 64-bit ids)
    n = 9

    def make():
        g, o = make_pair(n, topology="grid", latency_dist="constant", latency_mean_ms=4, n_values=1024, ring_cap=1024,
                         max_window=512, journal_cap_log2=20, max_endpoints=n + 8, calendar_slots=64, calendar_cap=4096)

        def scenario(s, body):
            c = s.add_endpoint("c0", O.KIND_SIM_CLIENT)
            ops, _ = random_broadcast_ops(n, [c], n_ticks=10, per_tick=12, seed=8)
            s.schedule(ops)
            h = s.add_endpoint("h0", O.KIND_HOST)
            for v in range(24):
                s.send(h, v % n, body("broadcast", msg_id=v + 1, p0=600 + v))
            s.run(2_000_000)                       # the broadcast_ok replies are in the wheel
            s.remove_endpoint(h)
            h2 = s.add_endpoint("h1", O.KIND_HOST)
            assert h2 == h                         # the slot is recycled
            for v in range(12):
                s.send(h2, (v * 5) % n, body("read", msg_id=100 + v))
            s.run(60_000_000)
            got = []
            while True:
                m = s.recv(h2, 0)
                if m is None:
                    break
                got.append((int(m["id"]), int(m["type"]), int(m["src"]), int(m["in_reply_to"])))
            return got
        return g, o, scenario
    return Case(make, False, node_sets=n, recv=True)


def workload(name, n=9, latency=0, services=(), ticks=8, per_tick=12, until_ms=40, **kw):
    from test_fuzz_parity import random_ops

    def make():
        g, o = make_pair(n, workload=name, latency_dist="constant", latency_mean_ms=latency, n_values=256,
                         ring_cap=1024, max_window=512, journal_cap_log2=20, max_endpoints=n + 12, calendar_slots=256,
                         calendar_cap=4096, **kw)

        def scenario(s, body):
            sv = {k: s.add_endpoint(k, O.KIND_SERVICE) for k in services}
            cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(3)]
            if name in ("g-set", "lin-kv"):
                for i in range(n):
                    s.send(cs[0], i, body("init", msg_id=9000 + i))
            if name == "lin-kv":
                rows = np.zeros(ticks * per_tick, dtype=O.OP_DTYPE)
                r2 = np.random.default_rng(5)
                for k in range(len(rows)):
                    r = rows[k]
                    r["time_ns"] = (2500 + k // per_tick * 7) * 1_000_000        # once a leader is elected
                    r["src"], r["dest"] = cs[k % 3], int(r2.integers(n))
                    b = r["body"]
                    b["flags"], b["msg_id"], b["p0"] = O.F_MSG_ID, k + 1, int(r2.integers(4))
                    kind = int(r2.integers(3))
                    b["type"] = (O.T["read"], O.T["write"], O.T["cas"])[kind]
                    b["p1"] = int(r2.integers(4)) | ((int(r2.integers(4)) << 32) if kind == 2 else 0)
                s.schedule(rows)
            else:
                s.schedule(random_ops(np.random.default_rng(2), n, cs, sv, name, 0, ticks, per_tick, [0] * 3))
            s.run(until_ms * 1_000_000)
            return s.client_replies()
        return g, o, scenario
    philox = latency > 0 or name == "lin-kv" or bool({"seq-kv", "lww-kv"} & set(services))
    return Case(make, philox, node_sets=n if name in ("broadcast", "g-set") else 0)


def txn_tree():
    from test_txn_tree import txn_ops
    from scenarios import ops_array
    n = 5

    def make():
        g, o = make_pair(n, workload="txn-list-append-tree", max_endpoints=n + 16, ring_cap=1024, max_window=512,
                         server_ring_cap=256, server_max_window=64, rpc_table=256, tree_ptrs=4096, journal_cap_log2=20,
                         seed=2 * 977)

        def scenario(s, body):
            s.add_endpoint("lin-kv", O.KIND_SERVICE)
            s.add_endpoint("lww-kv", O.KIND_SERVICE)
            cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(4)]
            s.schedule(ops_array([(0, cs[i % 4], i, "init", 1 + i // 4, 0) for i in range(n)]))
            s.schedule(txn_ops(np.random.default_rng(2), n, cs, 40, 30, 3, 40, [100] * 4))
            s.run(300 * 1_000_000)
            return s.client_replies()
        return g, o, scenario
    return Case(make, True)


def gen_clients():
    n, k = 9, 6

    def make():
        g, o = make_pair(n, topology="grid", n_values=1 << 12, ring_cap=1024, max_window=512, journal_cap_log2=20,
                         max_endpoints=n + 8)

        def scenario(s, body):
            s.add_gen_clients(k, interval_ns=2_000_000, time_limit_ns=40_000_000, read_permille=400,
                              timeout_ns=15_000_000, quiet_ns=20_000_000)
            s.run(70_000_000)
        return g, o, scenario
    return Case(make, True, node_sets=n, history=True)


SCENARIOS = {
    "bcast_compact": bcast(),
    "mixed_128": mixed(64, 65),
    "mixed_512": mixed(300, 211),
    "ring16": ring_wrap(16),
    "ring32": ring_wrap(32),
    "bcast_lat_const": bcast(latency=3),
    "bcast_lat_exp": bcast(latency=3, dist="exponential"),
    "loss": phases("loss_on_off"),
    "flaky": phases("flaky"),
    "drop": phases("drop_pair"),
    "partition": phases("partition_heal"),
    "remove_readd": remove_readd(),
    "echo": workload("echo"),
    "gset": workload("g-set", gset_interval_ms=7),
    "services": workload("broadcast", services=("lin-kv", "seq-kv", "lww-kv", "lin-tso")),
    "txn": workload("txn-list-append", services=("lin-kv",), n=5),
    "raft": workload("lin-kv", n=3, ticks=4, per_tick=6, until_ms=2800),
    "txn_tree": txn_tree(),
    "gen_clients": gen_clients(),
}

ORIGINS = ("id32", "id31", "ev32", "r15", "r31", "r32", "ring", "all")

# every origin for the broadcast paths; the boundaries most likely to be mishandled by the other programs
MATRIX = [(sc, og) for sc in ("bcast_compact", "bcast_lat_const") for og in ORIGINS]
MATRIX += [(sc, og) for sc in ("mixed_128", "mixed_512") for og in ("id32", "ev32", "r15", "ring", "all")]
MATRIX += [(sc, og) for sc in ("ring16", "ring32") for og in ("ring", "all")]
MATRIX += [(sc, og) for sc in ("bcast_lat_exp", "loss", "flaky", "drop", "partition", "remove_readd", "echo", "gset",
                                "services", "txn", "txn_tree", "gen_clients") for og in ("id32", "r15", "ring", "all")]
MATRIX += [("raft", og) for og in ("id32", "r15", "all")]


# ------------------------------------------------------------------------------------------- runs
class Probing:
    """Wraps an engine so that run(until) advances one round at a time (the same rounds: a run stops at the first
    round whose time reaches `until`) and records the ring counters at every stop."""

    def __init__(self, g):
        self.g = g
        self.stops = []

    def __getattr__(self, name):
        return getattr(self.g, name)

    def run(self, until_ns):
        while self.g.now < until_ns:
            self.g.step(1)
            self.stops.append(self.g.ring_counters())
        return 0


def run_case(case, origin, probe=False):
    """Runs the scenario on a fresh pair at `origin`; returns a dict of everything compared."""
    g, o, scenario = case.make()
    if origin:
        g.set_origin(**origin)
        o.set_origin(**origin)
    gp = Probing(g) if probe else g
    if case.compact:
        ring0 = g.ring_counters()
    rg, ro = both(gp, o, scenario)
    assert rg == ro
    out = {"g": g, "o": o, "stops": gp.stops if probe else [], "ret": rg}
    rc = g.ring_counters()
    out["rings"] = rc
    if case.compact:
        ev_o, bd_o = o.journal()
        want = oracle_gossip_sends(ev_o, bd_o, o.n_nodes)
        got = int((rc["ctail"] - ring0["ctail"]).astype(np.uint64).sum())      # claims since the origin, mod 2^32
        if case.compact == "eq":
            assert got == want, (got, want)
        else:
            assert got <= want, (got, want)
        out["compact"] = got
    if case.history:
        hg, ho = g.history(), o.history()
        assert len(hg) == len(ho) > 0
        for f in ("time_ns", "order", "client", "op", "type", "f", "error", "value"):
            assert np.array_equal(hg[f], ho[f]), f
        out["history"] = hg
    out["sets"] = [g.node_set(i).tolist() for i in range(case.node_sets)]
    assert out["sets"] == [o.node_set(i).tolist() for i in range(case.node_sets)]
    ev_g, bd_g = g.drain()
    ev_o, bd_o = o.journal()
    assert len(ev_g) == len(ev_o), (len(ev_g), len(ev_o))
    for f in ("event_id", "time_ns", "msg_id", "src", "dest"):
        if not np.array_equal(ev_g[f], ev_o[f]):
            bad = int(np.nonzero(ev_g[f] != ev_o[f])[0][0])
            raise AssertionError("journal field %s differs first at event %d: engine=%s oracle=%s" %
                                 (f, bad, ev_g[bad], ev_o[bad]))
    for f in ("type", "flags", "msg_id", "in_reply_to", "p0", "p1"):
        assert np.array_equal(bd_g[f], bd_o[f]), f
    assert np.array_equal(bd_g["id"], ev_g["msg_id"])
    out.update(ev=ev_g, bd=bd_g, stats=g.stats(), now=g.now, round=g.round)
    assert out["stats"] == o.stats() and out["now"] == o.now and out["round"] == o.round
    g.close()
    return out


_BASE = {}


def base_run(name, backend):
    """The scenario at origin 0, once per backend."""
    key = (name, backend)
    if key not in _BASE:
        _BASE[key] = run_case(SCENARIOS[name], None)
    return _BASE[key]


def inside_round_cut(ev, ids):
    """A position k in the :send events (ids = their message ids, or the event ids of all events) such that
    events k-1 and k belong to the same round and, where possible, the same sender: the cut between them is where
    an origin puts the 2^32 boundary.  Searched outward from the middle."""
    t, src = ev["time_ns"], ev["src"]
    n = len(ids)
    mid = n // 2
    fallback = None
    for d in range(n):
        for k in (mid - d, mid + d):
            if 1 <= k < n and t[k - 1] == t[k]:
                if src[k - 1] == src[k]:
                    return int(ids[k])
                if fallback is None:
                    fallback = int(ids[k])
    assert fallback is not None, "no round with two events"
    return fallback


def make_origin(kind, base):
    ev = base["ev"]
    sends = ev[(ev["event_id"] & RECV) == 0]
    id_cut = inside_round_cut(sends, sends["msg_id"])
    ev_cut = inside_round_cut(ev, ev["event_id"] & EVENT_MASK)
    rounds = base["round"]
    # rings: the busiest endpoint's counters cross 2^32 halfway through its traffic; the stride staggers the others
    tails = np.concatenate([base["rings"]["tail"], base["rings"]["ctail"]]).astype(np.int64)
    half = max(int(tails.max()) // 2, 1)
    ring = dict(ring_pos=(B32 - half) & 0xFFFFFFFF, ring_stride=3)
    one = {
        "id32": dict(msg_id=B32 - id_cut),
        "id31": dict(msg_id=B31 - id_cut),
        "ev32": dict(event_id=B32 - ev_cut),
        "r15": dict(round=B15 - rounds // 2),
        "r31": dict(round=B31 - rounds // 2),
        "r32": dict(round=B32 - rounds // 2),
        "ring": ring,
    }
    if kind == "all":
        return dict(msg_id=B32 - id_cut, event_id=B32 - ev_cut, round=B32 - rounds // 2, **ring)
    return one[kind]


def shifted(base, origin):
    """The origin-0 journal as the metamorphic relation predicts it at `origin`."""
    ev = base["ev"].copy()
    bd = base["bd"].copy()
    dm, de = np.uint64(origin.get("msg_id", 0)), np.uint64(origin.get("event_id", 0))
    ev["msg_id"] += dm
    bd["id"] += dm
    ev["event_id"] = ((ev["event_id"] & EVENT_MASK) + de) | (ev["event_id"] & RECV)
    return ev, bd


def check_crossed(kind, origin, res, base):
    ev = res["ev"]
    if "msg_id" in origin:
        b = B31 if kind == "id31" else B32
        ids = ev["msg_id"]
        assert int(ids.min()) < b <= int(ids.max())
        sends = ev[(ev["event_id"] & RECV) == 0]
        below = sends[sends["msg_id"] == b - 1]
        above = sends[sends["msg_id"] == b]
        assert len(below) == len(above) == 1 and below["time_ns"][0] == above["time_ns"][0]     # inside one round
    if "event_id" in origin:
        eids = ev["event_id"] & EVENT_MASK
        assert int(eids.min()) < B32 <= int(eids.max())
        k = int(np.nonzero(eids == B32)[0][0])
        assert ev["time_ns"][k - 1] == ev["time_ns"][k]
    if "round" in origin:
        b = {"r15": B15, "r31": B31}.get(kind, B32)
        assert origin["round"] < b < res["round"]
    if "ring_pos" in origin:
        # some counter wrapped while records or a window were open: tail < head numerically at a stop
        open_wrap = any(((st["tail"] < st["head"]) | (st["ctail"] < st["chead"])).any() for st in res["stops"])
        assert open_wrap, "no stop saw a ring counter wrapped past its head"


@pytest.mark.parametrize("name,kind", MATRIX)
def test_origin_parity(engine_backend, name, kind):
    case = SCENARIOS[name]
    base = base_run(name, engine_backend)
    origin = make_origin(kind, base)
    res = run_case(case, origin, probe="ring_pos" in origin)
    check_crossed(kind, origin, res, base)
    if case.compact == "eq":
        assert res["compact"] == base["compact"] > 0
    # metamorphic: the origin-0 run with its counters shifted
    if "round" in origin and case.philox:
        return
    ev, bd = shifted(base, origin)
    for f in ("event_id", "time_ns", "msg_id", "src", "dest"):
        assert np.array_equal(res["ev"][f], ev[f]), f
    for f in ("id", "type", "flags", "msg_id", "in_reply_to", "p0", "p1"):
        assert np.array_equal(res["bd"][f], bd[f]), f
    assert res["stats"] == base["stats"] and res["now"] == base["now"]
    assert res["round"] == base["round"] + origin.get("round", 0)
    assert res["sets"] == base["sets"]
    if case.recv:
        dm = origin.get("msg_id", 0)
        assert res["ret"] == [(r[0] + dm,) + r[1:] for r in base["ret"]]      # the host endpoint's message ids
    elif not case.history:
        assert res["ret"] == base["ret"]


# ------------------------------------------------------------------------------------------- streaming and files
def stream_pair(origin, n=25, level=1):
    g, o = make_pair(n, topology="grid", n_values=2048, ring_cap=1024, max_window=512, journal_cap_log2=18,
                     journal_level=level)
    g.set_origin(**origin)
    o.set_origin(**origin)
    cs = [g.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(3)]
    assert cs == [o.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(3)]
    ops, _ = random_broadcast_ops(n, cs, n_ticks=20, per_tick=40, seed=13)
    g.schedule(ops)
    o.schedule(ops)
    return g, o


@pytest.mark.parametrize("fmt", [4, 8, 12, 32])
def test_streamed_formats_across_the_id_and_event_boundaries(fmt):
    # ~25 k events: ids and event ids cross 2^32 about a third of the way in, and a MS_JFMT_4 decoder that
    # follows the stream from its start expands the receives on both sides of the crossing
    origin = dict(msg_id=B32 - 4321, event_id=B32 - 9876, round=B32 - 7)
    g, o = stream_pair(origin)
    got, heads = [], []

    def sink(info, rounds, ev):
        heads.append((info, rounds.copy()))
        got.append(ev.copy())

    g.run_streamed(60_000_000, sink, fmt=fmt, buf_events=2000, decode=True)
    o.run(60_000_000)
    ev_o, _ = o.journal()
    ev_g = np.concatenate(got)
    assert len(ev_g) == len(ev_o) > 20000 and len(heads) > 8
    for f in ("event_id", "time_ns", "msg_id", "src", "dest"):
        assert np.array_equal(ev_g[f], ev_o[f]), f
    assert g.stats() == o.stats() and g.now == o.now and g.round == o.round
    assert int(ev_g["msg_id"].min()) < B32 <= int(ev_g["msg_id"].max())
    assert int((ev_g["event_id"] & EVENT_MASK).min()) < B32 <= int((ev_g["event_id"] & EVENT_MASK).max())
    # headers: batches tile the event ids from the origin on; round rows carry the 64-bit bases
    first = origin["event_id"]
    straddle = False
    for info, rows in heads:
        assert info["first_event"] == first and info["format"] == fmt and not info["overflow"]
        first += info["n_events"]
        assert rows["ev_base"][0] <= info["first_event"] and np.all(np.diff(rows["ev_base"].astype(np.int64)) > 0)
        assert np.all(rows["round"] >= origin["round"])
        if fmt in (4, 8):
            assert np.all(rows["id_ref"] >= origin["msg_id"] - (1 << 30))
        straddle |= info["first_event"] < B32 < info["first_event"] + info["n_events"]
    assert first == origin["event_id"] + len(ev_o) and straddle


def test_format_12_near_its_47_bit_limit():
    # MS_JFMT_12 carries 47-bit ids: exact below 2^47, and a batch with a larger id reports overflow (the call
    # fails) instead of wrapping
    lim = 1 << 47
    g, o = stream_pair(dict(msg_id=lim - 30000))
    got = []
    with pytest.raises(Exception) as e:
        g.run_streamed(60_000_000, lambda info, rounds, ev: got.append(ev.copy()), fmt=12, buf_events=2000, decode=True)
    assert "cannot hold this batch" in str(e.value)
    o.run(60_000_000)
    ev_o, _ = o.journal()
    ev_g = np.concatenate(got)
    assert 0 < len(ev_g) < len(ev_o) and int(ev_g["msg_id"].max()) < lim
    for f in ("event_id", "time_ns", "msg_id", "src", "dest"):
        assert np.array_equal(ev_g[f], ev_o[f][:len(ev_g)]), f


@pytest.mark.parametrize("fmt", [8, 32])
def test_streamed_after_a_drain_across_the_boundary(fmt):
    # part of the journal is drained, the rest streamed: the stream's first batch starts where the drain ended
    origin = dict(msg_id=B32 - 7000, event_id=B32 - 14000)
    g, o = stream_pair(origin, level=2)
    g.run(2_000_000)
    ev_d, _ = g.drain()
    got = []
    g.run_streamed(60_000_000, lambda info, rounds, ev: got.append(ev.copy()), fmt=fmt, buf_events=3000, decode=True)
    o.run(60_000_000)
    ev_o, _ = o.journal()
    ev_g = np.concatenate([ev_d] + got)
    assert int(ev_d["msg_id"].max()) < B32 <= int(ev_g["msg_id"].max())
    for f in ("event_id", "time_ns", "msg_id", "src", "dest"):
        assert np.array_equal(ev_g[f], ev_o[f]), f


@cuda_only
def test_drain_into_pinned_memory_across_the_boundary():
    import torch
    origin = dict(msg_id=B32 - 5000, event_id=B32 - 7000)
    g, o = stream_pair(origin, level=2)
    g.run(60_000_000)
    o.run(60_000_000)
    ev_o, bd_o = o.journal()
    n = len(ev_o)
    ev = torch.empty(n * 32, dtype=torch.uint8, pin_memory=True)
    bd = torch.empty(n * 32, dtype=torch.uint8, pin_memory=True)
    got = 0
    while got < n:
        k = g.drain_into(ev.data_ptr() + got * 32, min(4096, n - got), bd.data_ptr() + got * 32)
        assert k > 0
        got += k
    ev_g = ev.numpy().view(O.EVENT_DTYPE)
    from maelstrom_b200._lib import JBODY_DTYPE
    bd_g = bd.numpy().view(JBODY_DTYPE)
    for f in ("event_id", "time_ns", "msg_id", "src", "dest"):
        assert np.array_equal(ev_g[f], ev_o[f]), f
    assert np.array_equal(bd_g["id"], ev_o["msg_id"]) and np.array_equal(bd_g["p0"], bd_o["p0"])
    assert int(ev_g["msg_id"].min()) < B32 <= int(ev_g["msg_id"].max())


def fressian_int(i):
    """FressianWriter.writeInt, restated from org.fressian's published encoding (not from ms_fressian.h): the
    packed form is chosen by the number of leading zeros of i (of ~i when negative)."""
    m = ~i if i < 0 else i
    lz = 64 - m.bit_length()

    def be(v, k):
        return (v & ((1 << (8 * k)) - 1)).to_bytes(k, "big")
    if lz <= 14:
        return bytes([0xF8]) + be(i, 8)                         # INT + 8 bytes
    if lz <= 22:
        return bytes([(0x7E + (i >> 48)) & 0xFF]) + be(i, 6)    # INT_PACKED_7_ZERO
    if lz <= 30:
        return bytes([(0x7A + (i >> 40)) & 0xFF]) + be(i, 5)    # INT_PACKED_6_ZERO
    if lz <= 38:
        return bytes([(0x76 + (i >> 32)) & 0xFF]) + be(i, 4)    # INT_PACKED_5_ZERO
    if lz <= 44:
        return bytes([(0x72 + (i >> 24)) & 0xFF]) + be(i, 3)    # INT_PACKED_4_ZERO
    if lz <= 51:
        return bytes([(0x68 + (i >> 16)) & 0xFF]) + be(i, 2)    # INT_PACKED_3_ZERO
    if lz <= 57 or i < -1:
        return bytes([(0x50 + (i >> 8)) & 0xFF]) + be(i, 1)     # INT_PACKED_2_ZERO
    return bytes([i & 0xFF])


@pytest.mark.parametrize("msg_id,event_id", [(B31 + 5, B31 + 9), (B32 + 7, B32 + 3), ((1 << 40) + 1, B32 - 1)])
def test_journal_files_with_wide_ids(tmp_path, msg_id, event_id):
    # the first event of the Fressian file byte for byte (layout of test_fressian_journal's hand fixture, with the
    # ids in their packed forms), every event through the reader, and the binary MSJ1 file record for record
    from fressian_reader import FressianReader
    from test_fressian_journal import HAND
    import maelstrom_b200 as mb
    rows = {}
    for kind in ("fressian", "bin"):
        g, o = make_pair(4, topology="line", n_values=16)
        g.set_origin(msg_id=msg_id, event_id=event_id)
        o.set_origin(msg_id=msg_id, event_id=event_id)
        path = str(tmp_path / ("0.fressian" if kind == "fressian" else "j.bin"))
        for s, body in ((g, mb.body), (o, O.body)):
            c = s.add_endpoint("c0")
            if s is g:
                s.journal_open(path)
            s.send(c, 1, body("broadcast", msg_id=1, p0=5))
            s.run(3_000_000)
            s.send(c, 2, body("read", msg_id=2))
            s.run(5_000_000)
            if s is g:
                s.journal_close()
        rows[kind] = open(path, "rb").read()
        ev_o, bd_o = o.journal()
        g.close()
    # HAND: STRUCTTYPE "ev" 4, event id 0 (offset 5), time 0, :send, STRUCTTYPE "msg" 4, message id 0 (offset 22) ...
    assert HAND[4] == 4 and HAND[5] == 0 and HAND[21] == 4 and HAND[22] == 0
    want = HAND[:5] + fressian_int(event_id) + HAND[6:22] + fressian_int(msg_id) + HAND[23:]
    data = rows["fressian"]
    assert data[:len(want)] == want, (data[:len(want)].hex(), want.hex())
    events = FressianReader(data).read_all()
    assert len(events) == len(ev_o) > 10
    for e, eo in zip(events, ev_o):
        assert e["id"] == int(eo["event_id"]) & ((1 << 63) - 1) and e["message"]["id"] == int(eo["msg_id"])
    binj = rows["bin"]
    hdr = np.frombuffer(binj[:16], dtype="<u4")
    assert hdr[0] == 0x314A534D and hdr[1] == 2
    rec = np.frombuffer(binj[16:], dtype=np.dtype([("ev", O.EVENT_DTYPE), ("bd", mb.engine.JBODY_DTYPE)]))
    for f in ("event_id", "time_ns", "msg_id", "src", "dest"):
        assert np.array_equal(rec["ev"][f], ev_o[f]), f


@pytest.mark.parametrize("msg_id", [B31 + 3, B32 + 11])
def test_json_envelope_ids_past_31_and_32_bits(msg_id):
    # ms_recv_json prints the network id as an exact JSON integer
    import maelstrom_b200 as mb
    g = mb.Sim(3, workload="echo", max_endpoints=8)
    g.set_origin(msg_id=msg_id)
    c = g.add_endpoint("c0")
    ids = [g.send(c, 0, mb.body("echo", msg_id=k + 1, p0=k)) for k in range(3)]
    assert ids == [msg_id, msg_id + 1, msg_id + 2]
    g.run(5_000_000)
    buf = C.create_string_buffer(4096)
    lines = []
    for _ in range(3):
        assert g.L.ms_recv_json(g.h, c, 0, buf, len(buf)) == 1
        lines.append(json.loads(buf.value.decode()))
    assert [m["id"] for m in lines] == [msg_id + 3, msg_id + 4, msg_id + 5]          # the echo_ok replies
    assert [m["body"]["in_reply_to"] for m in lines] == [1, 2, 3]
    g.close()


# ------------------------------------------------------------------------------------------- sharded emulator
@pytest.mark.parametrize("glue", [True, False], ids=["glue", "no_glue"])
@pytest.mark.parametrize("world", [2, 3, 4])
@pytest.mark.parametrize("kind", ["ring", "ids"])
def test_emulated_shards_at_an_origin(engine_backend, kind, world, glue, monkeypatch):
    # every shard takes the same origin and sets its own endpoints' ring counters; peer claims on wrapped counters
    # (48-B and compact rings of servers another shard owns) and the merged journal must match the oracle
    from test_emul_sharded import check_against_oracle, run_sharded_scenario
    if engine_backend != "emul":
        pytest.skip("emulated shards")
    if not glue:
        monkeypatch.setenv("MS_NO_GLUE", "1")
    n = 64
    origin = (dict(ring_pos=B32 - 150, ring_stride=5) if kind == "ring" else
              dict(msg_id=B32 - 9000, event_id=B32 - 18000, round=B32 - 9))
    kw = dict(topology="grid", n_values=1024, seed=29)
    counters = {}

    def scenario(s, body):
        s.set_origin(**origin)
        cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(3)]
        ops, _ = random_broadcast_ops(n, cs, n_ticks=6, per_tick=20, seed=33)
        s.schedule(ops)
        s.run(3_000_000)
        s.run(12_000_000)
        if is_engine(s):
            counters[s.cfg.shard_id] = s.ring_counters()

    sim_kw = dict(workload="broadcast", ring_cap=1024, max_window=512, journal_cap_log2=19, max_endpoints=n + 8, **kw)
    ev, st, now, rnd = run_sharded_scenario(world, n, sim_kw, scenario)
    o = O.Sim(n, workload=O.W_BROADCAST, **kw)
    check_against_oracle(o, scenario, ev, st, now, rnd)
    ev_o, bd_o = o.journal()
    start = np.array([(origin.get("ring_pos", 0) + e * origin.get("ring_stride", 0)) & 0xFFFFFFFF for e in range(n)],
                     dtype=np.uint32)
    from maelstrom_b200.sharded import shard_owner
    owners = np.array([shard_owner(e, n, world) for e in range(n)])
    claimed = sum((counters[r]["ctail"] - start)[owners == r].astype(np.uint64).sum() for r in range(world))
    assert int(claimed) == oracle_gossip_sends(ev_o, bd_o, n) > 1000
    if kind == "ring":
        assert any((counters[r]["ctail"] < start)[owners == r].any() for r in range(world))   # compact counters wrapped
    else:
        assert int(ev["msg_id"].min()) < B32 <= int(ev["msg_id"].max())


@pytest.mark.parametrize("world", [2, 3])
def test_emulated_shards_stream_across_the_boundary(engine_backend, world):
    # MS_JFMT_8 on shards is handed over as MS_JFMT_16 records: event id word + the id word relative to id_ref
    from test_emul_sharded import run_sharded_scenario
    import threading
    if engine_backend != "emul":
        pytest.skip("emulated shards")
    n = 36
    origin = dict(msg_id=B32 - 2500, event_id=B32 - 5000, ring_pos=B32 - 40, ring_stride=3)
    got, lock = {}, threading.Lock()

    def scenario(s, body):
        s.set_origin(**origin)
        cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(3)]
        ops, _ = random_broadcast_ops(n, cs, n_ticks=20, per_tick=12, seed=23)
        s.schedule(ops)
        if hasattr(s, "run_streamed"):
            mine = []

            def sink(info, rounds, ev):
                assert info["format"] == 16
                mine.append(ev.copy())
            s.run_streamed(25_000_000, sink, fmt=8, buf_events=1500, decode=True)
            with lock:
                got[s.cfg.shard_id] = np.concatenate(mine) if mine else np.zeros(0, dtype=O.EVENT_DTYPE)
        else:
            s.run(25_000_000)

    ev_left, st, now, rnd = run_sharded_scenario(
        world, n, dict(workload="broadcast", topology="grid", ring_cap=1024, max_window=512, journal_cap_log2=16,
                       max_endpoints=n + 8, n_values=2048), scenario)
    assert len(ev_left) == 0
    o = O.Sim(n, workload=O.W_BROADCAST, topology="grid", n_values=2048)
    scenario(o, O.body)
    ev_o, _ = o.journal()
    allv = np.concatenate([got[r] for r in range(world)])
    merged = allv[np.argsort(allv["event_id"] & EVENT_MASK, kind="stable")]
    assert len(merged) == len(ev_o) > 4000
    for f in ("event_id", "time_ns", "msg_id", "src", "dest"):
        assert np.array_equal(merged[f], ev_o[f]), f
    assert int(merged["msg_id"].min()) < B32 <= int(merged["msg_id"].max())
    assert st == o.stats() and now == o.now and rnd == o.round


# ------------------------------------------------------------------------------------------- GPU scale
@cuda_only
def test_three_phase_commit_at_a_round_origin():
    # more than 16 384 tickets: rounds are committed by k_commit_a / b / c; rounds, ids and events all cross 2^32
    n = 129 * 129
    g, o = make_pair(n, topology="grid", n_values=256, max_endpoints=n + 8, ring_cap=256, max_window=256,
                     journal_cap_log2=24, journal_level=1)
    origin = dict(round=B32 - 60, msg_id=B32 - 200_000, event_id=B32 - 400_000, ring_pos=B32 - 2, ring_stride=1)
    g.set_origin(**origin)
    o.set_origin(**origin)

    def scenario(s, body):
        c = s.add_endpoint("c0", O.KIND_SIM_CLIENT)
        for v in range(8):
            s.send(c, (v * 2039) % n, body("broadcast", msg_id=v + 1, p0=v))
        s.run(1_000_000)

    both(g, o, scenario)
    ev_g, _ = g.drain(bodies=False)
    ev_o, _ = o.journal()
    assert len(ev_g) == len(ev_o) > 700_000
    for f in ("event_id", "time_ns", "msg_id", "src", "dest"):
        assert np.array_equal(ev_g[f], ev_o[f]), f
    assert g.stats() == o.stats() and g.now == o.now and g.round == o.round > B32
    assert int(ev_g["msg_id"].min()) < B32 <= int(ev_g["msg_id"].max())
    assert [g.node_set(k).size for k in (0, n - 1)] == [8, 8]


@cuda_only
def test_bench_topology_heavy_windows_at_the_benchmark_id_range():
    # test_gpu_parity's bench-topology scenario (64 x 64 grid, windows in all four size classes, 30.8 M messages)
    # started where every bench.py run is: message ids across 2^32, event ids across 2^33
    from test_gpu_parity import hot_broadcast_ops
    n, V, ticks = 4096, 1280, 2
    g, o = make_pair(n, topology="grid", n_values=V * ticks + 8, max_endpoints=n + 8, ring_cap=8192, max_window=4096,
                     journal_cap_log2=26, journal_level=1)
    origin = dict(msg_id=B32 - 10 ** 7, event_id=(1 << 33) - 2 * 10 ** 7)
    g.set_origin(**origin)
    o.set_origin(**origin)

    def scenario(s, body):
        cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(4)]
        s.schedule(hot_broadcast_ops(n, cs, ticks, V, [10 * 64 + 10, 11 * 64 + 11, 40 * 64 + 50], 900, seed=77))
        s.run(ticks * 1_000_000)

    both(g, o, scenario)
    ev_g, _ = g.drain(bodies=False)
    ev_o, _ = o.journal()
    assert len(ev_g) == len(ev_o) == 2 * ticks * V * 12035
    for f in ("event_id", "time_ns", "msg_id", "src", "dest"):
        assert np.array_equal(ev_g[f], ev_o[f]), f
    assert g.stats() == o.stats() and g.round == o.round
    assert int(ev_g["msg_id"].min()) < B32 <= int(ev_g["msg_id"].max())
    eids = ev_g["event_id"] & EVENT_MASK
    assert int(eids.min()) < (1 << 33) <= int(eids.max())
    assert g.counters()["max_window"] == 2342
