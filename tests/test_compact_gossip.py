"""Server -> neighbor broadcast gossip in 16-B compact records (DESIGN.md 3.1): parity with the oracle at the
edges of that path, and an exact account of which messages took it.  The journal is the same whichever ring a
message went through, so every case also reads the servers' ring counters (Sim.ring_counters()) and checks
that the compact rings carried exactly the gossip they should:

- compact-eligible run (broadcast, constant latency 0, no loss, no endpoint removed, no message sent on a
  server's behalf, every server with <= 4 neighbors): compact records == the oracle's server -> server
  broadcast sends;
- otherwise: compact records <= those sends;
- echo / g-set, latency > 0 from the start, loss from the start or the total topology: no compact record.

Every case runs on the emulator ([emul], CPU suite) and on the H100 ([cuda])."""
import numpy as np
import pytest

import oracle_lib as O
from scenarios import (assert_same_journal, both, compact_delta, compact_total, make_pair, oracle_gossip_sends,
                       random_broadcast_ops)

pytestmark = pytest.mark.usefixtures("engine_backend")
cuda_only = pytest.mark.gpu


def is_engine(s):
    return hasattr(s, "ring_counters")


def check_accounting(g, o, expect):
    """expect: "eq", "le" or "zero" (see the module docstring); returns (compact records, oracle gossip)."""
    ev, bd = o.journal()
    want = oracle_gossip_sends(ev, bd, o.n_nodes)
    got = compact_total(g.ring_counters())
    if expect == "eq":
        assert got == want, (got, want)
    elif expect == "le":
        assert got <= want, (got, want)
    else:
        assert got == 0, got
    return got, want


def check_all(g, o, expect):
    res = check_accounting(g, o, expect)     # reads the oracle's journal before assert_same_journal drains the engine
    assert_same_journal(g, o)
    return res


# ------------------------------------------------------------------------------------------- accounting
@pytest.mark.parametrize("workload,topo,n,latency,p_loss,expect", [
    ("broadcast", "grid", 25, 0, 0.0, "eq"),
    ("broadcast", "line", 12, 0, 0.0, "eq"),
    ("broadcast", "tree3", 30, 0, 0.0, "eq"),
    ("broadcast", "grid", 25, 0, 0.1, "zero"),         # loss rolls need the general emission path
    ("broadcast", "grid", 25, 1, 0.0, "zero"),         # latency > 0: the timing wheel
    ("broadcast", "total", 8, 0, 0.0, "zero"),         # no neighbor table
    ("broadcast", "tree4", 40, 0, 0.0, "le"),          # degree 5: compact only for block-ordered windows
    ("echo", "grid", 9, 0, 0.0, "zero"),
    ("g-set", "grid", 9, 0, 0.0, "zero"),
])
def test_gossip_accounting(workload, topo, n, latency, p_loss, expect):
    from test_fuzz_parity import random_ops
    g, o = make_pair(n, workload=workload, topology=topo, latency_dist="constant", latency_mean_ms=latency,
                     p_loss=p_loss, n_values=1024, ring_cap=1024, max_window=512, journal_cap_log2=20,
                     max_endpoints=n + 8, gset_interval_ms=7)

    def scenario(s, body):
        cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(3)]
        if workload == "broadcast":
            ops, _ = random_broadcast_ops(n, cs, n_ticks=8, per_tick=25, seed=5)
        else:
            if workload == "g-set":
                for i in range(n):
                    s.send(cs[0], i, body("init", msg_id=9000 + i))
            ops = random_ops(np.random.default_rng(2), n, cs, {}, workload, 0, 8, 12, [0] * 3)
        s.schedule(ops)
        s.run((40 + 40 * latency) * 1_000_000)

    both(g, o, scenario)
    rc = g.ring_counters()
    got, want = check_all(g, o, expect)
    if workload != "broadcast":
        assert all(not v.any() for k, v in rc.items() if k.startswith("c"))   # no compact ring at all
    elif expect == "eq":
        assert want > 1000
        # ... and the servers' 48-B rings carried nothing but the clients' messages
        assert int(rc["tail"].astype(np.uint64).sum()) == 8 * 25
    elif expect == "le":
        assert got > 0                                 # light traffic: most windows are block-ordered


# ------------------------------------------------------------------------------------------- mixed windows
def mixed_window(k_g, k_f, **sizing):
    """5-node line: k_g values to server 2, one round, then k_f values to server 1.  Two rounds later server 1's
    window is k_f 48-B records from the client plus k_g compact records from server 2."""
    g, o = make_pair(5, topology="line", n_values=k_g + k_f + 8, ring_cap=8192, max_window=4096,
                     journal_cap_log2=20, **sizing)
    probes = []

    def scenario(s, body):
        c = s.add_endpoint("c0", O.KIND_SIM_CLIENT)
        for v in range(k_g):
            s.send(c, 2, body("broadcast", msg_id=v + 1, p0=v))
        s.step(1)
        for v in range(k_f):
            s.send(c, 1, body("broadcast", msg_id=k_g + v + 1, p0=k_g + v))
        for _ in range(2):
            s.step(1)
            if is_engine(s):
                probes.append(s.ring_counters())
        s.run(5_000_000)

    return g, o, scenario, probes


@pytest.mark.parametrize("k_g,k_f", [
    (64, 63), (64, 64), (64, 65),                      # sums around the 128 class boundary
    (0, 128), (0, 129), (128, 0), (129, 0),            # one part alone on either side of it
    (1, 127), (127, 1), (1, 128),
    (300, 211), (256, 256), (1, 512), (512, 1),        # ... around 512
    pytest.param(1000, 1047, marks=cuda_only), pytest.param(1024, 1024, marks=cuda_only),
    pytest.param(2047, 1, marks=cuda_only), pytest.param(0, 2048, marks=cuda_only),   # ... up to 2048
])
def test_mixed_window_at_class_boundaries(k_g, k_f):
    g, o, scenario, probes = mixed_window(k_g, k_f, server_ring_cap=4096, server_max_window=2048)
    both(g, o, scenario)
    # the round after the injection server 2 gossiped k_g values; the next, server 1 froze the mixed window
    p1 = probes[-1]
    assert int(p1["limit"][1] - p1["head"][1]) == k_f
    assert int(p1["climit"][1] - p1["chead"][1]) == k_g
    assert g.counters()["max_window"] == k_g + k_f
    check_all(g, o, "eq")


# ------------------------------------------------------------------------------------------- capacity errors
def test_window_overflow_is_decided_by_the_sum():
    # both parts fit server_ring_cap (256), their sum is server_max_window + 1
    import maelstrom_b200 as mb
    g = mb.Sim(5, topology="line", n_values=256, ring_cap=1024, max_window=512, server_ring_cap=256,
               server_max_window=128)
    c = g.add_endpoint("c0", O.KIND_SIM_CLIENT)
    for v in range(64):
        g.send(c, 2, mb.body("broadcast", msg_id=v + 1, p0=v))
    g.step(1)
    for v in range(65):
        g.send(c, 1, mb.body("broadcast", msg_id=65 + v, p0=64 + v))
    g.step(1)
    with pytest.raises(mb.SimError) as e:
        g.step(1)
    msg = str(e.value)
    assert "per-round window exceeds" in msg and "at endpoint 1 " in msg, msg
    # the error is latched: later calls report it again and run no round
    r = g.round
    with pytest.raises(mb.SimError) as e2:
        g.run(50_000_000)
    assert str(e2.value) == msg and g.round == r
    g.close()


def test_compact_ring_overflow_names_the_receiver():
    # servers 1 and 3 each gossip 40 new values to server 2 in the same round: 80 compact records for a ring of
    # 64 while every window (40) fits.  The claim overflows first (the window of 80 would only be seen the
    # round after), and the error names the receiving neighbor.
    import maelstrom_b200 as mb
    g = mb.Sim(5, topology="line", n_values=128, ring_cap=1024, max_window=64, server_ring_cap=64)
    c = g.add_endpoint("c0", O.KIND_SIM_CLIENT)
    for v in range(80):
        g.send(c, 1 if v < 40 else 3, mb.body("broadcast", msg_id=v + 1, p0=v))
    g.step(1)
    with pytest.raises(mb.SimError) as e:
        g.step(1)
    msg = str(e.value)
    assert "inbox ring overflow" in msg and "at endpoint 2 " in msg, msg
    r = g.round
    with pytest.raises(mb.SimError) as e2:
        g.step(1)
    assert str(e2.value) == msg and g.round == r
    g.close()


# ------------------------------------------------------------------------------------------- wrap
def both_rings_wrap(cap):
    """5-node line with server rings of `cap` records, values to servers 1 and 3 every round for 40 * cap / 16
    rounds: every compact ring wraps several times.  Returns (engine, oracle, scenario, probes); probes collects
    the engine's ring counters after each of those rounds."""
    n, rounds = 5, 40 * cap // 16
    g, o = make_pair(n, topology="line", n_values=4096, ring_cap=1024, max_window=256, server_ring_cap=cap,
                     journal_cap_log2=20)
    rng = np.random.default_rng(cap)
    # up to cap / 4 values per round to servers 1 and 3: server 2's compact ring holds a window of up to cap / 2
    # (from both) plus as many new claims
    plan = [(int(rng.integers(1, cap // 4 + 1)), int(rng.integers(1, cap // 4 + 1))) for _ in range(rounds)]
    probes = []

    def scenario(s, body):
        c = s.add_endpoint("c0", O.KIND_SIM_CLIENT)
        v = 0
        for a, b in plan:
            for dest, k in ((1, a), (3, b)):
                for _ in range(k):
                    s.send(c, dest, body("broadcast", msg_id=v + 1, p0=v))
                    v += 1
            s.step(1)
            if is_engine(s):
                probes.append(s.ring_counters())
        s.run(5_000_000)

    return g, o, scenario, probes


@pytest.mark.parametrize("cap", [16, 32])
def test_windows_wrap_on_both_rings(cap):
    # small server rings, many rounds: every compact ring wraps several times, and frozen windows straddle the
    # wrap of the 48-B ring and of the compact ring of the same server in the same round
    n = 5
    g, o, scenario, probes = both_rings_wrap(cap)
    both(g, o, scenario)

    def straddles(head, limit):
        return (limit - head) > 0 and (head % cap) + (limit - head) > cap

    both_rings = [(k, e) for k, p in enumerate(probes) for e in range(n)
                  if straddles(int(p["head"][e]), int(p["limit"][e])) and straddles(int(p["chead"][e]), int(p["climit"][e]))]
    assert both_rings, "no round froze a window across the wrap of both rings"
    assert all(int(t) > 4 * cap for t in probes[-1]["ctail"]), probes[-1]["ctail"]
    check_all(g, o, "eq")


# ------------------------------------------------------------------------------------------- fast path off / on
def phase_scenario(change, n=16):
    """Grid traffic in phases; between phase 1 and 2 the run stops with compact records pending and `change` is
    applied.  Returns (scenario, marks): marks collects, per phase boundary, the engine's ring counters or the
    oracle's journal length."""
    marks = []
    steps = []

    def mark(s):
        marks.append(s.ring_counters() if is_engine(s) else len(s.journal()[0]))

    def scenario(s, body):
        cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(3)]
        ops, nv = random_broadcast_ops(n, cs, n_ticks=12, per_tick=20, seed=9)
        s.schedule(ops)
        s.run(3_000_000)
        if is_engine(s):                               # (the engine runs first: the oracle takes as many steps)
            for _ in range(16):                        # stop between rounds with gossip in flight
                s.step(1)
                steps.append(1)
                rc = s.ring_counters()
                if (rc["ctail"] != rc["climit"]).any():
                    break
            else:
                raise AssertionError("no round left compact records pending")
        else:
            s.step(len(steps))
        mark(s)
        change(s, body, cs)
        s.run(7_000_000)
        mark(s)
        if change.__name__ in ("loss_on_off", "partition_heal"):
            s.set_loss(0.0) if change.__name__ == "loss_on_off" else s.heal()
            s.run(13_000_000)
            mark(s)
        s.run(40_000_000)

    return scenario, marks


def remove_client(s, body, cs):
    s.remove_endpoint(cs[2])


def loss_on_off(s, body, cs):
    s.set_loss(0.2)


def flaky(s, body, cs):
    s.flaky()


def partition_heal(s, body, cs):
    s.partition([i % 2 for i in range(16)])


def drop_pair(s, body, cs):
    s.drop(5, 6)
    s.drop(9, 5)


@pytest.mark.parametrize("change", [remove_client, loss_on_off, flaky, partition_heal, drop_pair],
                         ids=lambda f: f.__name__)
def test_fast_path_switches_with_records_in_flight(change):
    g, o = make_pair(16, topology="grid", n_values=1024, ring_cap=1024, max_window=512, journal_cap_log2=20,
                     max_endpoints=24)
    scenario, marks = phase_scenario(change)
    both(g, o, scenario)
    ev, bd = o.journal()
    eng = [m for m in marks if isinstance(m, dict)]
    orc = [m for m in marks if not isinstance(m, dict)]
    assert (eng[0]["ctail"] != eng[0]["climit"]).any()   # the change came with compact records pending
    # gossip per phase: the oracle's sends between two marks, the engine's compact claims between the same two
    orc_gossip = [oracle_gossip_sends(ev[a:b], bd[a:b], 16) for a, b in zip(orc, orc[1:] + [len(ev)])]
    eng_compact = [int(compact_delta(b, a).astype(np.uint64).sum()) for a, b in zip(eng, eng[1:])]
    eng_compact.append(compact_total(g.ring_counters()) - compact_total(eng[-1]))
    assert orc_gossip[0] > 0
    name = change.__name__
    if name == "remove_client":
        assert eng_compact == [0, 0]                      # any removal turns the fast path off for good
    elif name == "loss_on_off":
        assert eng_compact[0] == 0 < orc_gossip[0]        # loss rolls: the general path
        assert eng_compact[1:] == orc_gossip[1:]          # loss back to 0: all gossip compact again
    elif name == "flaky":
        assert eng_compact == [0, 0]
    else:                                               # cuts at dequeue do not change the sending side
        assert eng_compact == orc_gossip
        c = g.counters()
        st = o.stats()["all"]
        assert c["partition_drops"] == st["send-count"] - st["recv-count"] > 0   # no loss, nothing left in flight
    exact = name in ("partition_heal", "drop_pair")
    check_all(g, o, "eq" if exact else "le")


def test_send_on_a_servers_behalf_falls_back_for_one_window():
    # a host message with a server as src turns the fast path off for the CTA of its receiver, in the round that
    # receiver consumes it, and for nobody else
    n = 16
    g, o = make_pair(n, topology="grid", n_values=1024, ring_cap=1024, max_window=512, journal_cap_log2=20,
                     max_endpoints=24)
    marks = []

    def scenario(s, body):
        cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(3)]
        ops, nv = random_broadcast_ops(n, cs, n_ticks=6, per_tick=20, seed=4)
        s.schedule(ops)
        s.run(2_000_000)
        mid = s.send(0, 6, body("broadcast", p0=701))            # a fresh value, on server 0's behalf
        for _ in range(4):
            marks.append((s.ring_counters() if is_engine(s) else len(s.journal()[0]), mid))
            s.step(1)
        marks.append((s.ring_counters() if is_engine(s) else len(s.journal()[0]), mid))
        s.run(30_000_000)

    both(g, o, scenario)
    ev, bd = o.journal()
    eng = [m for m, _ in marks[:5]]
    orc = [m for m, _ in marks[5:]]
    mid = marks[5][1]
    assert mid == marks[0][1]
    recv = (ev["event_id"] & np.uint64(O.RECV_BIT)) != 0
    not_injected = ev["msg_id"] != mid                # the host's message itself travels in a 48-B ring
    fell_back = 0
    for k in range(4):
        a, b = orc[k], orc[k + 1]
        sl = slice(a, b)
        want = oracle_gossip_sends(ev[sl][not_injected[sl]], bd[sl][not_injected[sl]], n)
        got = int(compact_delta(eng[k + 1], eng[k]).astype(np.uint64).sum())
        if (recv[sl] & (ev["msg_id"][sl] == mid)).any():             # the round server 6 consumed it
            ev6 = ev[sl][(ev["src"][sl] == 6) & ~recv[sl]]
            bd6 = bd[sl][(ev["src"][sl] == 6) & ~recv[sl]]
            lost = oracle_gossip_sends(ev6, bd6, n)
            assert lost > 0 and got == want - lost, (got, want, lost)
            fell_back += 1
        else:
            assert got == want, (k, got, want)
    assert fell_back == 1
    check_all(g, o, "le")


# ------------------------------------------------------------------------------------------- ordering fallbacks
@pytest.mark.parametrize("topo,n,n_clients", [("tree4", 40, 8), ("grid", 16, 70)])
@pytest.mark.parametrize("jlevel", [1, 2])
def test_bitonic_fallback_with_a_compact_part(topo, n, n_clients, jlevel):
    # a hot node: hundreds of client messages per round interleave in its 48-B ring (many sender blocks, or blocks
    # that overlap) next to its neighbors' compact gossip; level 1 takes the shared-memory :recv path, level 2
    # the rebuilding one
    per_tick, ticks = 600, 2
    g, o = make_pair(n, topology=topo, n_values=per_tick * ticks + 8, ring_cap=8192, max_window=4096,
                     journal_cap_log2=21, journal_level=jlevel, max_endpoints=n + n_clients + 4)

    def scenario(s, body):
        cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(n_clients)]
        rows = np.zeros(ticks * per_tick, dtype=O.OP_DTYPE)
        r2 = np.random.default_rng(3)
        for k in range(len(rows)):
            r = rows[k]
            r["time_ns"] = (k // per_tick) * 1_000_000
            r["src"] = cs[k % n_clients]
            r["dest"] = 0 if r2.integers(2) else int(r2.integers(n))
            b = r["body"]
            b["type"], b["flags"], b["msg_id"], b["p0"] = O.T["broadcast"], O.F_MSG_ID, k + 1, k
        s.schedule(rows)
        s.run((ticks + 3) * 1_000_000)

    both(g, o, scenario)
    c = g.counters()
    assert c["fallback_sorts"] > 0
    got, want = check_accounting(g, o, "eq" if topo == "grid" else "le")
    assert got > 0
    if jlevel == 2:
        assert_same_journal(g, o)
    else:
        ev_g, _ = g.drain(bodies=False)
        ev_o, _ = o.journal()
        assert len(ev_g) == len(ev_o)
        for f in ("event_id", "time_ns", "msg_id", "src", "dest"):
            assert np.array_equal(ev_g[f], ev_o[f]), f
        assert g.stats() == o.stats() and g.now == o.now and g.round == o.round


# ------------------------------------------------------------------------------------------- streaming
@pytest.mark.parametrize("fmt", [4, 8, 12, 32])
def test_streamed_journal_of_compact_traffic(fmt):
    n = 25
    g, o = make_pair(n, topology="grid", n_values=2048, ring_cap=1024, max_window=512, journal_cap_log2=18,
                     journal_level=1)
    cs = [g.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(3)]
    assert cs == [o.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(3)]
    ops, _ = random_broadcast_ops(n, cs, n_ticks=20, per_tick=40, seed=13)
    g.schedule(ops)
    o.schedule(ops)
    got = []
    g.run_streamed(60_000_000, lambda info, rounds, ev: got.append(ev.copy()), fmt=fmt, buf_events=2000, decode=True)
    o.run(60_000_000)
    ev_o, _ = o.journal()
    ev_g = np.concatenate(got)
    assert len(ev_g) == len(ev_o) > 20000
    for f in ("event_id", "time_ns", "msg_id", "src", "dest"):
        assert np.array_equal(ev_g[f], ev_o[f]), f
    assert g.stats() == o.stats() and g.now == o.now and g.round == o.round
    check_accounting(g, o, "eq")
