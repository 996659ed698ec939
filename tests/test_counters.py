"""The g-counter and pn-counter workloads (MS_W_G_COUNTER / MS_W_PN_COUNTER, DESIGN.md 2.16): demo/ruby/pn_counter.rb's
CRDT node on the device, in blocks of g servers, driven by the closed-loop counter clients (ms_add_gen_clients).
Journal, stats, time, the history and every node's counter must equal the oracle twin's (tests/native/counter_oracle.cpp);
the node's rules are read back from host-driven exchanges; and the checker of workload/pn_counter.clj, restated below,
passes on every block once the replication has had its quiet period, fails on stale final reads, and runs under the
device partition nemesis.  [emul] = the kernel sources on the CPU SIMT emulator, [cuda] = an H100."""
import numpy as np
import pytest

import counter_oracle_lib as CT
import oracle_lib as O
from scenarios import assert_same_journal, both, ops_array

pytestmark = pytest.mark.usefixtures("engine_backend")
MS = 1_000_000
INVOKE, OK, FAIL, INFO = 0, 1, 2, 3
TIMEOUT = 0xFFFF
READ, ADD = 1, 14                                                # MS_HF_READ, MS_HF_COUNTER_ADD
MERGE, MERGE_OK = 80, 81
HIST_FIELDS = ("time_ns", "order", "client", "op", "type", "f", "error", "value")
RECV = np.uint64(1 << 63)
WORKLOADS = ("g-counter", "pn-counter")


def counter_pair(workload, n, n_clients, g=0, interval_ms=200, **kw):
    """(engine, oracle twin) of n counter nodes in blocks of g, with room for n_clients clients"""
    import maelstrom_b200 as mb
    args = dict(latency_dist="constant", latency_mean_ms=0, max_endpoints=n + n_clients + 8, ring_cap=256,
                max_window=256, server_ring_cap=64, server_max_window=64, raft_group=g, journal_cap_log2=20,
                calendar_slots=64, calendar_cap=max(1024, 8 * n_clients), gset_interval_ms=interval_ms)
    args.update(kw)
    shared = {k: args[k] for k in ("latency_dist", "latency_mean_ms", "p_loss", "raft_group", "seed",
                                   "gset_interval_ms") if k in args}
    return mb.Sim(n, workload=workload, **args), CT.Sim(n, workload, **shared)


def start(s, n):
    """an init sink (index n), every node initialised in the first round"""
    sink = s.add_endpoint("c99999", O.KIND_SIM_CLIENT)
    s.schedule(ops_array([(0, sink, i, "init", 1 + i, 0) for i in range(n)]))
    s.run(5 * MS)
    return sink


def clients_scenario(n, n_clients, limit, quiet, jump=False, stretches=1, **client_kw):
    kw = dict(interval_ns=10 * MS, time_limit_ns=limit, quiet_ns=quiet)
    kw.update(client_kw)
    until = limit + quiet + kw.get("timeout_ns", 0) + 300 * MS

    def scenario(s, body):
        if jump and hasattr(s, "idle_jump"):                # the oracle ticks: it is the reference for both runs
            s.idle_jump()
        start(s, n)
        s.add_gen_clients(n_clients, **kw)
        hist = []
        for k in range(1, stretches + 1):
            s.run(5 * MS + (until - 5 * MS) * k // stretches)
            hist.append(s.history())
        return np.concatenate(hist)
    return scenario


def node_state(s, n):
    return [tuple(a.tolist() for a in s.counter_state(i)) for i in range(n)]


def same_history(hg, ho):
    assert len(hg) == len(ho) > 0
    for f in HIST_FIELDS:
        assert np.array_equal(hg[f], ho[f]), f


def run_pair(workload, n, n_clients, scenario, **kw):
    """both sides of one scenario: everything observable must be equal; returns (engine, history, events, bodies)"""
    g, o = counter_pair(workload, n, n_clients, **kw)
    hg, ho = both(g, o, scenario)
    same_history(hg, ho)
    ev, bd = assert_same_journal(g, o)
    assert node_state(g, n) == node_state(o, n)
    o.close()
    return g, hg, ev, bd


# ------------------------------------------------------------------------------------------- the checker
def acceptable(adds):
    """pn_counter.clj:79-125: the sum of the :ok adds, and for every :info add either with or without it.  `adds` =
    [(delta, ok)]; returns the acceptable set as sorted, disjoint closed ranges [lo, hi]"""
    ranges = [(sum(d for d, ok in adds if ok),) * 2]
    for d, ok in adds:
        if ok:
            continue
        both_ = sorted(ranges + [(lo + d, hi + d) for lo, hi in ranges])
        ranges = [both_[0]]
        for lo, hi in both_[1:]:                                    # open ranges (lo - 1, hi + 1) merge when adjacent
            if lo <= ranges[-1][1] + 1:
                ranges[-1] = (ranges[-1][0], max(ranges[-1][1], hi))
            else:
                ranges.append((lo, hi))
    return ranges


def signed(v):
    return int(np.array(v, dtype=np.uint32).view(np.int32))


def check(h, n_nodes, first, group, final_from):
    """the checker per block of `group` servers (0 = one block): client c is on node (c - first) mod n_nodes; a final
    read is a read invoked at or after final_from.  An add without a completion counts as :info.  Returns {block:
    (valid, final read values, acceptable ranges, definite sum)}"""
    group = group or n_nodes
    recs = h[h["client"] != 0xFFFFFFFF]                            # not the nemesis's
    blocks = {}
    done = {}
    for r in recs[recs["type"] != INVOKE]:
        done[(int(r["client"]), int(r["op"]))] = r
    for r in recs[recs["type"] == INVOKE]:
        c = int(r["client"])
        b = (c - first) % n_nodes // group
        adds, finals = blocks.setdefault(b, ([], []))
        end = done.get((c, int(r["op"])))
        if r["f"] == ADD:
            adds.append((signed(r["value"]), end is not None and end["type"] == OK))
        elif r["f"] == READ and int(r["time_ns"]) >= final_from and end is not None and end["type"] == OK:
            finals.append(signed(end["value"]))
    out = {}
    for b, (adds, finals) in blocks.items():
        ranges = acceptable(adds)
        valid = all(any(lo <= v <= hi for lo, hi in ranges) for v in finals)
        out[b] = (valid, finals, ranges, sum(d for d, ok in adds if ok))
    return out


def test_checker_restatement():
    assert acceptable([(3, True), (2, True)]) == [(5, 5)]
    assert acceptable([(3, True), (2, False), (-1, False)]) == [(2, 5)]
    assert acceptable([(0, True), (10, False), (20, False)]) == [(0, 0), (10, 10), (20, 20), (30, 30)]
    assert acceptable([(4, False), (-4, False)]) == [(-4, -4), (0, 0), (4, 4)]


# ------------------------------------------------------------------------------------------- parity
@pytest.mark.parametrize("workload", WORKLOADS)
@pytest.mark.parametrize("dist", ["constant", "exponential"])
def test_parity_with_the_counter_oracle_twin_jump_off_and_on(workload, dist):
    n, n_clients, g = 6, 12, 3
    net = dict(latency_dist="constant", latency_mean_ms=0) if dist == "constant" else \
        dict(latency_dist="exponential", latency_mean_ms=20, p_loss=0.1)
    client = dict(timeout_ns=150 * MS) if dist == "exponential" else {}   # timeouts under loss, stale replies
    runs = []
    for jump in (False, True):
        sc = clients_scenario(n, n_clients, 1000 * MS, 500 * MS, jump, stretches=2, **client)
        eng, h, ev, bd = run_pair(workload, n, n_clients, sc, g=g, **net)
        runs.append((h, ev, bd, eng.stats(), eng.now, eng.round, node_state(eng, n)))
        if jump:
            assert eng.counters()["rounds"] < eng.round                     # the jump skipped rounds
        eng.close()
    (h0, ev0, bd0, *rest0), (h1, ev1, bd1, *rest1) = runs
    assert h0.tobytes() == h1.tobytes() and ev0.tobytes() == ev1.tobytes() and bd0.tobytes() == bd1.tobytes()
    assert rest0 == rest1
    done = h0[h0["type"] != INVOKE]
    assert np.count_nonzero((done["f"] == ADD) & (done["type"] == OK)) > 50
    assert np.count_nonzero((done["f"] == READ) & (done["type"] == OK)) > 50
    deltas = [signed(v) for v in h0[(h0["type"] == INVOKE) & (h0["f"] == ADD)]["value"]]
    assert set(deltas) == (set(range(-5, 5)) if workload == "pn-counter" else set(range(0, 5)))
    sends = (ev0["event_id"] & RECV) == 0
    merges = sends & (bd0["type"] == MERGE)
    assert np.count_nonzero(merges) > 20 and np.all(ev0["dest"][merges] // g == ev0["src"][merges] // g)
    if dist == "exponential":
        assert np.count_nonzero(done["error"] == TIMEOUT) > 0
    else:
        assert np.count_nonzero(done["error"] == TIMEOUT) == 0


def test_default_read_shares():
    import maelstrom_b200 as mb
    for workload, share in (("g-counter", 667), ("pn-counter", 500)):
        n, nc = 2, 40
        with mb.Sim(n, workload=workload, max_endpoints=64, gset_interval_ms=100) as s:
            start(s, n)
            s.add_gen_clients(nc, interval_ns=5 * MS, time_limit_ns=2000 * MS, quiet_ns=200 * MS)
            s.run(2500 * MS)
            h = s.history()
            inv = h[(h["type"] == INVOKE) & (h["time_ns"] < 2000 * MS)]
            got = 1000 * np.count_nonzero(inv["f"] == READ) / len(inv)
            assert abs(got - share) < 40, (workload, got)


# ------------------------------------------------------------------------------------------- the node, host-driven
def host_scenario(s, body):
    """one host client against node n0 of a block of three: adds with and without msg_id, negative deltas, reads,
    merge_ok and a stray reply (ignored), a second init; then the replication carries n0's counter to n1 and n2"""
    c = s.add_endpoint("c1", O.KIND_CLIENT)
    got = []

    def rpc(b, expect=True, to=0):
        s.send(c, to, b)
        m = s.recv(c, 50 * MS)
        assert (m is not None) == expect
        if m is not None:
            got.append(tuple(int(m[k]) for k in ("type", "flags", "in_reply_to", "p0", "p1")))
    for i in range(3):
        rpc(body("init", msg_id=1), to=i)
    rpc(body("add", msg_id=2, p0=5))
    rpc(body("add", msg_id=3, p0=-3 & 0xFFFFFFFF))
    rpc(body("add", p0=4))                                                    # no msg_id: no in_reply_to
    rpc(body("read", msg_id=4))
    rpc(body("read"))
    rpc(body(MERGE_OK, msg_id=5), expect=False)                              # crdt.rb:36-38: ignored
    rpc(body("add_ok", in_reply_to=3), expect=False)                         # a reply: no callback, ignored
    rpc(body("add", msg_id=6, in_reply_to=9, p0=100), expect=False)          # anything with in_reply_to is a reply
    rpc(body("read", msg_id=8), to=1)                                        # n0's adds are not replicated yet
    before = node_state(s, 3)
    rpc(body("init", msg_id=7))                                              # a second init restarts the task
    s.run(s.now + 250 * MS)                                                  # one replication run later
    rpc(body("read", msg_id=9), to=1)
    rpc(body("read", msg_id=10), to=2)
    return got, before, node_state(s, 3)


@pytest.mark.parametrize("workload", WORKLOADS)
def test_node_rules_host_driven(workload):
    g, o = counter_pair(workload, 3, 0, g=3)
    rg, ro = both(g, o, host_scenario)
    assert rg == ro
    got, before, after = rg
    R = O.F_REPLY
    init_ok, add_ok, read_ok = O.T["init_ok"], O.T["add_ok"], O.T["read_ok"]
    assert got == [
        (init_ok, R, 1, 0, 0), (init_ok, R, 1, 0, 0), (init_ok, R, 1, 0, 0),
        (add_ok, R, 2, 0, 0), (add_ok, R, 3, 0, 0), (add_ok, 0, 0, 0, 0),
        (read_ok, R, 4, 0, 6), (read_ok, 0, 0, 0, 6),
        (read_ok, R, 8, 0, 0),
        (init_ok, R, 7, 0, 0),
        (read_ok, R, 9, 0, 6), (read_ok, R, 10, 0, 6)]
    assert before[0] == ([9, 0, 0], [3, 0, 0]) and before[1] == ([0, 0, 0], [0, 0, 0])
    assert after == [([9, 0, 0], [3, 0, 0])] * 3
    # merges go to the other block members in index order, carry the run, and their merge_ok has no in_reply_to
    ev, bd = assert_same_journal(g, o)
    sends = (ev["event_id"] & RECV) == 0
    m = sends & (bd["type"] == MERGE)
    assert np.count_nonzero(m) >= 6
    src0 = m & (ev["src"] == 0)
    assert ev["dest"][src0][:2].tolist() == [1, 2] and bd["p1"][src0][:2].tolist() == [1, 1]
    assert np.all(bd["flags"][m] == 0)
    mo = sends & (bd["type"] == MERGE_OK) & (ev["src"] < 3)
    assert np.count_nonzero(mo) == np.count_nonzero(~sends & (bd["type"] == MERGE)) > 0   # every merge received is answered
    assert np.all(bd["flags"][mo] == 0) and np.all(bd["in_reply_to"][mo] == 0)
    g.close()
    o.close()


def test_forged_merge_latches_the_snapshot_error():
    import maelstrom_b200 as mb
    for src_is_server, p1 in ((False, 1), (True, 77)):
        with mb.Sim(3, workload="pn-counter", max_endpoints=16) as s:
            c = s.add_endpoint("c1", O.KIND_CLIENT)
            s.send(1 if src_is_server else c, 0, mb.body(MERGE, p1=p1))
            with pytest.raises(mb.SimError) as e:
                s.run(3 * MS)
            assert e.value.code == -3 and "merge" in str(e.value)


def crash_scenario(s, body):
    """n0 gets a type it has no handler for: it crashes, its clients time out as :info, reads included; n1 serves on"""
    start(s, 2)
    c = s.add_endpoint("c77777", O.KIND_CLIENT)
    s.send(c, 0, body("echo", msg_id=1))
    s.run(10 * MS)
    s.add_gen_clients(4, interval_ns=20 * MS, time_limit_ns=600 * MS, timeout_ns=100 * MS, quiet_ns=300 * MS)
    s.run(1200 * MS)
    return s.history(), node_state(s, 2)


@pytest.mark.parametrize("workload", WORKLOADS)
def test_unknown_type_crashes_the_node(workload):
    g, o = counter_pair(workload, 2, 4, g=2, interval_ms=100)
    (hg, sg), (ho, so) = both(g, o, crash_scenario)
    same_history(hg, ho)
    assert sg == so
    ev, bd = assert_same_journal(g, o)
    host, first = 3, 4                                                # 2 nodes, the sink, the host client
    done = hg[hg["type"] != INVOKE]
    on0 = (done["client"] - first) % 2 == 0
    assert np.all((done["type"][on0] == INFO) & (done["error"][on0] == TIMEOUT))
    assert np.count_nonzero(on0 & (done["f"] == READ)) > 0
    assert np.all(done["type"][~on0] == OK)
    crash_t = int(ev["time_ns"][(ev["src"] == host) & (ev["dest"] == 0)][0])
    assert not np.any(((ev["event_id"] & RECV) == 0) & (ev["src"] == 0) & (ev["time_ns"] > crash_t))   # never sends
    g.close()
    o.close()


def test_refusals():
    import maelstrom_b200 as mb
    with pytest.raises(mb.SimError) as e:
        mb.Sim(2000, workload="pn-counter", raft_group=1025)
    assert "at most 1024 servers per block" in str(e.value)
    with pytest.raises(mb.SimError) as e:
        mb.Sim(1025, workload="g-counter")                            # g = 0: one block of every server
    assert "at most 1024 servers per block" in str(e.value)
    with mb.Sim(1024, workload="g-counter", max_endpoints=1100):
        pass
    with pytest.raises(mb.SimError) as e:
        mb.Sim(4, workload="pn-counter", n_shards=2, shard_id=0)
    assert "one GPU" in str(e.value)
    with mb.Sim(10, workload="pn-counter", raft_group=5) as s:
        for bad in (2, 10):
            with pytest.raises(mb.SimError) as e:
                s.nemesis(time_limit_ns=100 * MS, group=bad)
            assert e.value.code == -2
        s.nemesis(time_limit_ns=100 * MS, group=5)
    with mb.Sim(3, workload="kafka") as s:
        with pytest.raises(mb.SimError) as e:
            s.counter_state(0)
        assert e.value.code == -2 and "ms_counter_state" in str(e.value)
    with mb.Sim(3, workload="pn-counter") as s:
        with pytest.raises(mb.SimError):
            s.counter_state(3)
        with pytest.raises(mb.SimError):
            s.raft_state(0)
        with pytest.raises(mb.SimError):
            s.add_kv_clients(6, interval_ns=MS, time_limit_ns=MS, key_period_ns=MS)


# ------------------------------------------------------------------------------------------- the checker on runs
def checked_run(workload, quiet_ms, seed=0x5EED):
    n, n_clients, g = 6, 24, 3
    limit = 1500 * MS
    sc = clients_scenario(n, n_clients, limit, quiet_ms * MS, interval_ns=20 * MS)
    eng, h, _, _ = run_pair(workload, n, n_clients, sc, g=g, seed=seed, interval_ms=400)   # runs at 1, 401, .. 1601 ms
    eng.close()
    return h, check(h, n, n + 1, g, limit + quiet_ms * MS)


@pytest.mark.parametrize("workload", WORKLOADS)
def test_checker_passes_after_the_quiet_period_and_has_teeth(workload):
    h, res = checked_run(workload, 1000)                              # quiet = 2.5 replication intervals
    assert len(res) == 2
    for valid, finals, ranges, definite in res.values():
        assert valid and len(finals) == 12 and all(v == definite for v in finals)
        assert ranges == [(definite, definite)]                       # no loss: every add is :ok
    # one altered final read fails a passing history
    reads = np.nonzero((h["type"] == OK) & (h["f"] == READ) & (h["time_ns"] >= 2500 * MS))[0]
    bad = h.copy()
    bad["value"][reads[3]] = np.uint32((signed(bad["value"][reads[3]]) + 7) & 0xFFFFFFFF)
    assert sum(not v[0] for v in check(bad, 6, 7, 3, 2500 * MS).values()) == 1
    # final reads less than one replication interval after the mix are stale
    _, stale = checked_run(workload, 1)
    assert not all(v[0] for v in stale.values())


# ------------------------------------------------------------------------------------------- the nemesis
NEM_N, NEM_G, NEM_C = 10, 5, 20


def nemesis_scenario(s, make):
    start(s, NEM_N)
    s.add_gen_clients(NEM_C, interval_ns=20 * MS, time_limit_ns=1500 * MS, quiet_ns=1000 * MS)
    R = make(s)
    for t in (800, 2000, 2800):
        R.run(t * MS)
    return node_state(s, NEM_N)


@pytest.mark.parametrize("workload", WORKLOADS)
def test_nemesis_blocks_equal_the_host_driven_twins_and_pass_the_checker(workload):
    from test_nemesis import twins
    kw = dict(workload=workload, raft_group=NEM_G, max_endpoints=NEM_N + NEM_C + 8, gset_interval_ms=200,
              latency_dist="exponential", latency_mean_ms=5, calendar_slots=64)
    nem = dict(time_limit_ns=1500 * MS, interval_ns=150 * MS, start_ns=5 * MS, now0=5 * MS)   # installed after the inits
    oracle = lambda: CT.Sim(NEM_N, workload, raft_group=NEM_G, gset_interval_ms=200,   # noqa: E731
                            latency_dist="exponential", latency_mean_ms=5, seed=0x4D41454C)
    oa, rows, ops = twins(NEM_N, NEM_G, nemesis_scenario, nem, oracle=oracle, **kw)
    assert len(rows) > 4 and len({r[6] for r in rows}) == 2
    h = oa["hist"]
    res = check(h, NEM_N, NEM_N + 1, NEM_G, 2500 * MS)
    assert len(res) == 2
    for valid, finals, ranges, definite in res.values():
        assert valid and len(finals) == NEM_C // 2, (finals, ranges)
    sends = (oa["ev"]["event_id"] & RECV) == 0
    assert oa["stats"]["servers"]["send-count"] > oa["stats"]["servers"]["recv-count"]   # the cuts dropped merges
    assert np.count_nonzero(sends & (oa["bd"]["type"] == MERGE)) > 50


# ------------------------------------------------------------------------------------------- scale (GPU)
SCALE_N, SCALE_C, SCALE_G = 4095, 8190, 5
SCALE = dict(ring_cap=64, max_window=64, server_ring_cap=64, server_max_window=32, journal_cap_log2=24,
             calendar_slots=64, max_endpoints=SCALE_N + SCALE_C + 8, raft_group=SCALE_G, gset_interval_ms=1000)
SCALE_LIMIT, SCALE_QUIET = 3130, 2500
SCALE_STRETCHES = (1000, 2000, 3000, 4500, SCALE_LIMIT + SCALE_QUIET + 400)


def scale_scenario(hist):
    def scenario(s, body):
        sink = s.add_endpoint("c99999", O.KIND_SIM_CLIENT)               # 32 init_ok a millisecond fit its ring
        s.schedule(ops_array([((i % 128) * MS, sink, i, "init", 1 + i, 0) for i in sorted(range(SCALE_N), key=lambda i: i % 128)]))
        s.run(130 * MS)
        s.add_gen_clients(SCALE_C, interval_ns=100 * MS, time_limit_ns=SCALE_LIMIT * MS, quiet_ns=SCALE_QUIET * MS)
        for t in SCALE_STRETCHES:
            s.run(t * MS)
            hist.append(s.history())
        return [tuple(a.tolist() for a in s.counter_state(i)) for i in range(0, SCALE_N, 7)]
    return scenario


@pytest.fixture(scope="module")
def scale_oracle():
    """the oracle twin's run of the scale scenario, once for the tests below"""
    o = CT.Sim(SCALE_N, "pn-counter", raft_group=SCALE_G, gset_interval_ms=1000)
    ho = []
    state = scale_scenario(ho)(o, None)
    return o, state, np.concatenate(ho)


def scale_engine(**kw):
    import maelstrom_b200 as mb
    return mb.Sim(SCALE_N, workload="pn-counter", **dict(SCALE, **kw))


def check_scale(h):
    res = check(h, SCALE_N, SCALE_N + 1, SCALE_G, (SCALE_LIMIT + SCALE_QUIET) * MS)
    assert len(res) == SCALE_N // SCALE_G
    for valid, finals, ranges, definite in res.values():
        assert valid and len(finals) == 2 * SCALE_G


@pytest.mark.gpu
def test_scale_819_blocks_8190_clients(engine_backend, scale_oracle):
    if engine_backend != "cuda":
        pytest.skip("4095 counter nodes: GPU only")
    o, state, ho = scale_oracle
    g = scale_engine()
    hg = []
    assert scale_scenario(hg)(g, None) == state
    hg = np.concatenate(hg)
    same_history(hg, ho)
    assert len(hg) > 20 * SCALE_C
    assert_same_journal(g, o)
    check_scale(hg)
    g.close()


@pytest.mark.gpu
def test_scale_streamed_with_the_history_drained_between_stretches(engine_backend, scale_oracle):
    if engine_backend != "cuda":
        pytest.skip("4095 counter nodes: GPU only")
    from test_stream_overlap import Streamer, compare
    o, state, ho = scale_oracle
    g = scale_engine(journal_level=1)
    s = Streamer(g, 8, 1 << 22, drain_between=True)
    hg = []
    assert scale_scenario(hg)(s, None) == state
    hg = np.concatenate(hg)
    same_history(hg, ho)
    compare(s.journal(), o, g)
    assert len(s.batches) > 3
    check_scale(hg)
    g.close()


def wide_scenario(s, body):
    """one block of 1024: latency = replication interval, so a run's merges land with the previous run's merge_oks"""
    start(s, 1024)
    s.add_gen_clients(8, interval_ns=10 * MS, time_limit_ns=200 * MS, quiet_ns=80 * MS)
    s.run(330 * MS)
    return s.history(), [tuple(a.tolist() for a in s.counter_state(i)) for i in (0, 7, 500, 1023)]


@pytest.mark.gpu
def test_one_block_of_1024_with_merge_windows_above_1023(engine_backend):
    if engine_backend != "cuda":
        pytest.skip("1024-wide block: GPU only")
    import maelstrom_b200 as mb
    kw = dict(latency_dist="constant", latency_mean_ms=100, gset_interval_ms=100)
    g = mb.Sim(1024, workload="pn-counter", max_endpoints=1100, ring_cap=4096, max_window=4096, server_ring_cap=4096,
               server_max_window=4096, journal_cap_log2=25, calendar_slots=256, calendar_cap=1 << 14, **kw)
    o = CT.Sim(1024, "pn-counter", **kw)
    (hg, sg), (ho, so) = both(g, o, wide_scenario)
    same_history(hg, ho)
    assert sg == so and len(sg[0][0]) == 1024
    assert_same_journal(g, o)
    assert g.counters()["max_window"] > 1023
    g.close()
    o.close()
