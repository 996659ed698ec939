"""The txn-rw-register workload (MS_W_TXN_RW, DESIGN.md 2.17): demo/clojure/txn_rw_register_hat.clj's node on the
device, in blocks of g servers, driven by the closed-loop txn clients (ms_add_txn_rw_clients).  Journal, stats, time,
the history and every node's log and state must equal the oracle twin's (tests/native/txn_rw_oracle.cpp, which keeps
the Clojure's unreplicated map); the node's rules are read back from host-driven exchanges; and the read-committed
analyses Elle runs on this history, restated below with the availability checker, pass on device runs and fail on
edited ones.  [emul] = the kernel sources on the CPU SIMT emulator, [cuda] = an H100."""
import numpy as np
import pytest

import oracle_lib as O
import txn_rw_oracle_lib as RW
from scenarios import assert_same_journal, both, ops_array

pytestmark = pytest.mark.usefixtures("engine_backend")
MS = 1_000_000
INVOKE, OK, FAIL, INFO = 0, 1, 2, 3
TIMEOUT = 0xFFFF
TXN, TXN_OK, REPLICATE, REPLICATE_ACK = 60, 61, 90, 91
HIST_FIELDS = ("time_ns", "order", "client", "op", "type", "f", "error", "node", "index", "base", "ops", "reads")
RECV = np.uint64(1 << 63)


def rw_pair(n, n_clients, g=0, **kw):
    """(engine, oracle twin) of n txn-rw-register nodes in blocks of g, with room for n_clients clients"""
    import maelstrom_b200 as mb
    args = dict(latency_dist="constant", latency_mean_ms=0, max_endpoints=n + n_clients + 8, ring_cap=256,
                max_window=256, server_ring_cap=64, server_max_window=64, raft_group=g, journal_cap_log2=20,
                calendar_slots=64, calendar_cap=max(1024, 8 * n_clients), gset_interval_ms=100)
    args.update(kw)
    shared = {k: args[k] for k in ("latency_dist", "latency_mean_ms", "p_loss", "raft_group", "seed", "gset_interval_ms",
                                   "txn_rw_keys", "txn_rw_log_cap") if k in args}
    return mb.Sim(n, workload="txn-rw-register", **args), RW.Sim(n, **shared)


def start(s, n):
    """an init sink (index n), every node initialised in the first round"""
    sink = s.add_endpoint("c99999", O.KIND_SIM_CLIENT)
    s.schedule(ops_array([(0, sink, i, "init", 1 + i, 0) for i in range(n)]))
    s.run(5 * MS)
    return sink


def clients_scenario(n, n_clients, limit, jump=False, stretches=1, **client_kw):
    kw = dict(interval_ns=10 * MS, time_limit_ns=limit, key_period_ns=200 * MS, key_count=3)
    kw.update(client_kw)
    until = limit + kw.get("timeout_ns", 0) + 300 * MS

    def scenario(s, body):
        if jump and hasattr(s, "idle_jump"):                # the oracle ticks: it is the reference for both runs
            s.idle_jump()
        start(s, n)
        s.add_txn_rw_clients(n_clients, **kw)
        hist = []
        for k in range(1, stretches + 1):
            s.run(5 * MS + (until - 5 * MS) * k // stretches)
            hist.append(s.txn_rw_history())
        return np.concatenate(hist)
    return scenario


def node_state(s, nodes):
    out = []
    for i in nodes:
        lamport, n, val, ts = s.txn_rw_state(i)
        out.append((lamport, n, val.tobytes(), ts.tobytes(), s.txn_rw_log(i).tobytes()))
    return out


def same_history(hg, ho):
    assert len(hg) == len(ho) > 0
    for f in HIST_FIELDS:
        assert np.array_equal(hg[f], ho[f]), f


def run_pair(n, n_clients, scenario, **kw):
    """both sides of one scenario: everything observable must be equal; returns (engine, history, events, bodies)"""
    g, o = rw_pair(n, n_clients, **kw)
    hg, ho = both(g, o, scenario)
    same_history(hg, ho)
    ev, bd = assert_same_journal(g, o)
    assert node_state(g, range(n)) == node_state(o, range(n))
    for i in range(n):                                   # the twin's unreplicated map: every txn served, none acked
        assert o.unreplicated(i)[0] == g.txn_rw_state(i)[1]
    o.close()
    return g, hg, ev, bd


# ------------------------------------------------------------------------------------------- the checker
def mops(ops, base, reads=None):
    """[(write, key, value)] of a record's micro-ops: a write's value is base + i, a read's reads[i] (None: unknown)"""
    out = []
    for i in range(4):
        op = (int(ops) >> (16 * i)) & 0xFFFF
        if op & 0x8000:
            w = bool(op & 0x4000)
            out.append((w, op & 0x3FFF, int(base) + i if w else (None if reads is None else int(reads[i]))))
    return out


def txns(h):
    """{(client, op): (outcome, micro-ops)}: the invocations with their completions (None: none)"""
    done = {(int(r["client"]), int(r["op"])): r for r in h[h["type"] != INVOKE]}
    out = {}
    for r in h[h["type"] == INVOKE]:
        k = (int(r["client"]), int(r["op"]))
        end = done.get(k)
        typ = None if end is None else int(end["type"])
        out[k] = (typ, mops(r["ops"], r["base"], end["reads"] if typ == OK else None))
    return out


def check(h):
    """Elle's read-committed analyses on a history with unique writes per key (wfr-keys), and the availability checker
    with :availability :total (checker.clj:6-30).  Returns the set of anomaly names found"""
    t = txns(h)
    bad = set()
    writer, final = {}, {}                               # (key, value) -> txn; txn's last write per key
    for k, (typ, ms) in t.items():
        for w, key, v in ms:
            if w:
                writer[(key, v)] = k
                final[(k, key)] = v
    edges = {k: set() for k, (typ, _) in t.items() if typ == OK}
    for k, (typ, ms) in t.items():
        if typ != OK:
            continue
        seen = {}                                        # internal consistency: the txn's own prior state of a key
        for w, key, v in ms:
            if w:
                seen[key] = v
                continue
            if key in seen and seen[key] != v:
                bad.add("internal")
            seen[key] = v
            if v == 0:
                continue
            src = writer.get((key, v))
            if src is None:
                bad.add("garbage-read")
                continue
            if src == k:
                continue
            if t[src][0] == FAIL:
                bad.add("G1a")
            if final[(src, key)] != v:
                bad.add("G1b")
            if src in edges:
                edges[src].add(k)                        # wr
        first = {}                                       # ww: a write follows a read of the same key in the txn
        for w, key, v in ms:
            if not w and key not in first and v:
                first[key] = v
            elif w and key in first:
                src = writer.get((key, first[key]))
                if src is not None and src != k and src in edges:
                    edges[src].add(k)
    if has_cycle(edges):
        bad.add("G1c")
    if any(typ != OK for typ, _ in t.values()):
        bad.add("availability")
    return bad


def has_cycle(edges):
    color = dict.fromkeys(edges, 0)
    for root in edges:
        if color[root]:
            continue
        stack = [(root, iter(edges[root]))]
        color[root] = 1
        while stack:
            v, it = stack[-1]
            nxt = next(it, None)
            if nxt is None:
                color[v] = 2
                stack.pop()
            elif color.get(nxt) == 1:
                return True
            elif color.get(nxt) == 0:
                color[nxt] = 1
                stack.append((nxt, iter(edges[nxt])))
    return False


def synthetic(rows):
    """a history from (client, op, type, ops, base, reads) rows, one invocation before each completion"""
    import maelstrom_b200 as mb
    h = np.zeros(2 * len(rows), dtype=mb._lib.TXN_RW_HIST_DTYPE)
    for j, (c, op, typ, ops, base, reads) in enumerate(rows):
        for r, t in ((h[2 * j], INVOKE), (h[2 * j + 1], typ)):
            r["client"], r["op"], r["type"], r["ops"], r["base"] = c, op, t, ops, base
        h[2 * j + 1]["reads"] = reads
    return h


def mop(write, key):
    return 0x8000 | (0x4000 if write else 0) | key


def test_checker_restatement():
    w0, r0, w1, r1 = mop(1, 0), mop(0, 0), mop(1, 1), mop(0, 1)
    ok = [(1, 1, OK, w0 | w0 << 16, 10, [0] * 4), (2, 1, OK, r0, 20, [11, 0, 0, 0])]
    assert check(synthetic(ok)) == set()
    assert check(synthetic([ok[0], (2, 1, OK, r0, 20, [10, 0, 0, 0])])) == {"G1b"}      # T1's first write of key 0
    assert check(synthetic([(1, 1, FAIL, w0, 10, [0] * 4), (2, 1, OK, r0, 20, [10, 0, 0, 0])])) == {"G1a", "availability"}
    assert check(synthetic([(1, 1, OK, r0, 10, [99, 0, 0, 0])])) == {"garbage-read"}
    assert check(synthetic([(1, 1, OK, w0 | r0 << 16, 10, [0, 5, 0, 0])])) == {"internal", "garbage-read"}
    cyc = [(1, 1, OK, w0 | r1 << 16, 10, [0, 20, 0, 0]), (2, 1, OK, w1 | r0 << 16, 20, [0, 10, 0, 0])]
    assert check(synthetic(cyc)) == {"G1c"}                                                # wr both ways
    assert check(synthetic([(1, 1, INFO, w0, 10, [0] * 4)])) == {"availability"}


# ------------------------------------------------------------------------------------------- parity
@pytest.mark.parametrize("dist", ["constant", "exponential"])
def test_parity_with_the_txn_rw_oracle_twin_jump_off_and_on(dist):
    n, n_clients, g = 6, 12, 3
    net = dict(latency_dist="constant", latency_mean_ms=0) if dist == "constant" else \
        dict(latency_dist="exponential", latency_mean_ms=20, p_loss=0.1)
    client = dict(timeout_ns=150 * MS) if dist == "exponential" else {}   # timeouts under loss, stale replies
    runs = []
    for jump in (False, True):
        sc = clients_scenario(n, n_clients, 1000 * MS, jump, stretches=2, **client)
        eng, h, ev, bd = run_pair(n, n_clients, sc, g=g, **net)
        runs.append((h, ev, bd, eng.stats(), eng.now, eng.round, node_state(eng, range(n))))
        if jump:
            assert eng.counters()["rounds"] < eng.round                     # the jump skipped rounds
        eng.close()
    (h0, ev0, bd0, *rest0), (h1, ev1, bd1, *rest1) = runs
    assert h0.tobytes() == h1.tobytes() and ev0.tobytes() == ev1.tobytes() and bd0.tobytes() == bd1.tobytes()
    assert rest0 == rest1
    done = h0[h0["type"] != INVOKE]
    assert np.count_nonzero(done["type"] == OK) > 150
    assert set(len(mops(o, 0)) for o in h0["ops"]) == {1, 2, 3, 4}
    sends = (ev0["event_id"] & RECV) == 0
    reps = sends & (bd0["type"] == REPLICATE)
    assert np.count_nonzero(reps) > 20 and np.all(ev0["dest"][reps] == ev0["src"][reps] // g * g + (ev0["src"][reps] % g == 0))
    acks = sends & (bd0["type"] == REPLICATE_ACK)
    assert np.count_nonzero(acks) > 0 and np.all(ev0["dest"][acks] // g == ev0["src"][acks] // g)
    if dist == "exponential":
        assert np.count_nonzero(done["error"] == TIMEOUT) > 0
    else:
        assert np.count_nonzero(done["type"] != OK) == 0
        assert check(h0) == set()


# ------------------------------------------------------------------------------------------- the node, host-driven
K1, K2 = 5, 9


def host_scenario(s, body):
    """one host client against a block of two: a txn before init, the inits, txns with and without msg_id, an unknown
    type, a stray reply, a second init; then the replication task runs at 100 and 200 ms"""
    c = s.add_endpoint("c1", O.KIND_CLIENT)
    got = []

    def rpc(b, expect=True, to=0):
        s.send(c, to, b)
        m = s.recv(c, 40 * MS)
        assert (m is not None) == expect
        if m is not None:
            got.append(tuple(int(m[k]) for k in ("type", "flags", "in_reply_to", "p0", "p1")))
    rpc(body("txn", msg_id=1, p0=500, p1=mop(1, K1)), expect=False)                # blocks on the node-id promise
    rpc(body("init", msg_id=1), to=0)
    rpc(body("init", msg_id=1), to=1)
    ops = mop(0, K1) | mop(1, K1) << 16 | mop(0, K1) << 32 | mop(1, K2) << 48       # nil, write 101, read 101, write 103
    rpc(body("txn", msg_id=2, p0=100, p1=ops))
    rpc(body("txn", msg_id=3, p0=200, p1=mop(0, K1) | mop(0, K2) << 16))            # serial: reads 101, 103
    rpc(body("txn", p0=300, p1=mop(1, K2)))                                           # no msg_id: no in_reply_to
    rpc(body("echo", msg_id=5))                                                       # error 10, serves on
    rpc(body("txn_ok", in_reply_to=2), expect=False)                                  # a reply: ignored
    rpc(body("init", msg_id=6))                                                       # a second init changes nothing
    s.run(250 * MS)
    return got, node_state(s, (0, 1))


def test_node_rules_host_driven():
    g, o = rw_pair(2, 0, g=2)
    rg, ro = both(g, o, host_scenario)
    assert rg == ro
    got, state = rg
    R = O.F_REPLY
    assert got == [(O.T["init_ok"], R, 1, 0, 0), (O.T["init_ok"], R, 1, 0, 0),
                   (TXN_OK, R, 2, 0, 0), (TXN_OK, R, 3, 1, 1), (TXN_OK, 0, 0, 2, 2),
                   (O.T["error"], R, 5, 10, 0), (O.T["init_ok"], R, 6, 0, 0)]
    log = g.txn_rw_log(0)
    assert log["lamport"].tolist() == [0, 1, 2] and log["base"].tolist() == [100, 200, 300]
    assert log["reads"].tolist() == [[0, 0, 101, 0], [101, 103, 0, 0], [0, 0, 0, 0]]
    lamport, n, val, ts = g.txn_rw_state(0)
    assert (lamport, n, int(val[K1]), int(ts[K1]), int(val[K2]), int(ts[K2])) == (3, 3, 101, 0, 300, 2)
    ev, bd = assert_same_journal(g, o)
    sends = (ev["event_id"] & RECV) == 0
    rep = sends & (bd["type"] == REPLICATE)
    assert ev["time_ns"][rep].tolist() == [100 * MS, 200 * MS]                       # t0 + 100 k ms, none from n1
    assert ev["src"][rep].tolist() == [0, 0] and ev["dest"][rep].tolist() == [1, 1] and bd["p0"][rep].tolist() == [3, 3]
    assert np.all(bd["flags"][rep] == 0)
    ack = sends & (bd["type"] == REPLICATE_ACK)
    assert ev["src"][ack].tolist() == [1, 1] and ev["dest"][ack].tolist() == [0, 0] and bd["p0"][ack].tolist() == [3, 3]
    # n1 learned no write, only lamport += 3 per replicate; n0's acks removed nothing
    assert g.txn_rw_state(1)[:2] == (6, 0) and not g.txn_rw_state(1)[2].any()
    assert g.txn_rw_state(0)[:2] == (3, 3) and o.unreplicated(0) == (3, 1)
    g.close()
    o.close()


def test_key_range_and_full_log_latch():
    import maelstrom_b200 as mb
    for kw, p1, n_txns, text in ((dict(txn_rw_keys=16), mop(0, 16), 1, "value"),
                                 (dict(txn_rw_log_cap=2), mop(1, 3), 3, "reserved[3]")):
        with mb.Sim(2, workload="txn-rw-register", max_endpoints=16, **kw) as s:
            c = s.add_endpoint("c1", O.KIND_CLIENT)
            s.send(c, 0, mb.body("init", msg_id=1))
            s.run(3 * MS)
            for k in range(n_txns):
                s.send(c, 0, mb.body("txn", msg_id=2 + k, p0=10, p1=p1))
            with pytest.raises(mb.SimError) as e:
                s.run(10 * MS)
            assert e.value.code == -3 and text in str(e.value)


def test_refusals():
    import maelstrom_b200 as mb
    for n, g in ((4, 1), (64, 64), (40, 0), (6, 4)):
        with pytest.raises(mb.SimError) as e:
            mb.Sim(n, workload="txn-rw-register", raft_group=g)
        assert "blocks of 2 to 32 servers" in str(e.value)
    with mb.Sim(32, workload="txn-rw-register", max_endpoints=64):
        pass
    with pytest.raises(mb.SimError) as e:
        mb.Sim(4, workload="txn-rw-register", n_shards=2, shard_id=0)
    assert "one GPU" in str(e.value)
    with pytest.raises(mb.SimError):
        mb.Sim(4, workload="txn-rw-register", txn_rw_keys=16385)
    kw = dict(interval_ns=MS, time_limit_ns=MS, key_period_ns=MS)
    with mb.Sim(3, workload="kafka") as s:
        with pytest.raises(mb.SimError) as e:
            s.add_txn_rw_clients(3, **kw)
        assert e.value.code == -2
        with pytest.raises(mb.SimError):
            s.txn_rw_log(0)
    with mb.Sim(3, workload="txn-rw-register", max_endpoints=64, txn_rw_keys=8) as s:
        for bad in (dict(n_clients=4), dict(min_len=3, max_len=2), dict(max_len=5), dict(min_len=0),
                    dict(key_count=0), dict(key_count=9), dict(key_period_ns=0)):
            args = dict(kw, n_clients=3)
            args.update(bad)
            with pytest.raises(mb.SimError) as e:
                s.add_txn_rw_clients(**args)
            assert e.value.code == -2, bad
        with pytest.raises(mb.SimError):
            s.add_gen_clients(3, interval_ns=MS, time_limit_ns=MS)
        with pytest.raises(mb.SimError):
            s.add_kv_clients(6, **kw)
        s.add_txn_rw_clients(3, **kw)
        with pytest.raises(mb.SimError):
            s.add_txn_rw_clients(3, first_name=100, **kw)                   # a second time
        with pytest.raises(mb.SimError):
            s.add_kafka_clients(3, interval_ns=MS, time_limit_ns=MS)
        with pytest.raises(mb.SimError):
            s.txn_rw_state(3)
        with pytest.raises(mb.SimError):
            s.raft_state(0)
        with pytest.raises(mb.SimError):
            s.counter_state(0)
        for bad in (2, 1):
            with pytest.raises(mb.SimError):
                s.nemesis(time_limit_ns=100 * MS, group=bad)


# ------------------------------------------------------------------------------------------- the checker on runs
def test_checker_passes_on_device_runs_and_fails_on_edited_ones():
    n, n_clients, g = 4, 16, 2
    sc = clients_scenario(n, n_clients, 1500 * MS, key_count=2)
    eng, h, _, _ = run_pair(n, n_clients, sc, g=g)
    eng.close()
    assert check(h) == set()
    ok = np.nonzero(h["type"] == OK)[0]
    # an intermediate read: another txn through the same node reads a value its writer overwrote in the same txn
    inter = None
    for j in ok:
        ms = mops(h["ops"][j], h["base"][j])
        keys = [k for w, k, _ in ms if w]
        dup = [k for k in set(keys) if keys.count(k) > 1]
        if dup:
            inter = (j, dup[0], next(v for w, k, v in ms if w and k == dup[0]))
            break
    assert inter is not None
    j, key, v = inter
    reader = next(r for r in ok if r != j and h["node"][r] == h["node"][j] and
                  any(not w and k == key for w, k, _ in mops(h["ops"][r], 0)))
    slot = next(i for i in range(4) if (int(h["ops"][reader]) >> (16 * i)) & 0xC000 == 0x8000 and
                (int(h["ops"][reader]) >> (16 * i)) & 0x3FFF == key)
    bad = h.copy()
    bad["reads"][reader][slot] = v
    assert "G1b" in check(bad)
    # a wr cycle: two txns whose first micro-ops become reads of each other's first write
    a, b = [r for r in ok if mops(h["ops"][r], 0)[0][0]][:2]
    ka, kb = 100, 101                                                       # keys no other txn touches
    bad = h.copy()
    for r, own, other, other_base in ((a, ka, kb, int(h["base"][b])), (b, kb, ka, int(h["base"][a]))):
        ops = int(bad["ops"][r]) & ~0xFFFF | mop(1, own)                    # micro-op 0 writes `own`
        last = len(mops(ops, 0))
        if last < 4:
            ops |= mop(0, other) << (16 * last)
        else:
            ops = ops & ~(0xFFFF << 48) | mop(0, other) << 48
            last = 3
        bad["ops"][r] = ops
        bad["reads"][r][last] = other_base
    for r in (a, b):                                                       # the invocations carry the same ops
        inv = np.nonzero((bad["type"] == INVOKE) & (bad["client"] == bad["client"][r]) & (bad["op"] == bad["op"][r]))[0]
        bad["ops"][inv] = bad["ops"][r]
    assert "G1c" in check(bad)


# ------------------------------------------------------------------------------------------- the demo's shape
NEM_N, NEM_G, NEM_C = 8, 2, 16


def nemesis_scenario(s, make):
    start(s, NEM_N)
    s.add_txn_rw_clients(NEM_C, interval_ns=20 * MS, time_limit_ns=1500 * MS, key_period_ns=300 * MS, key_count=2)
    R = make(s)
    hist = []
    for t in (800, 1600, 2000):
        R.run(t * MS)
        hist.append(s.txn_rw_history())
    return np.concatenate(hist).tobytes(), node_state(s, range(NEM_N))


def test_demo_blocks_of_two_under_the_partition_nemesis():
    """the demo's shape (core.clj:113-126): :node-count 2 under partitions, read committed and total availability"""
    import maelstrom_b200 as mb
    from test_nemesis import twins
    kw = dict(workload="txn-rw-register", raft_group=NEM_G, max_endpoints=NEM_N + NEM_C + 8,
              latency_dist="exponential", latency_mean_ms=5, calendar_slots=64)
    nem = dict(time_limit_ns=1500 * MS, interval_ns=150 * MS, start_ns=5 * MS, now0=5 * MS)   # installed after the inits
    oracle = lambda: RW.Sim(NEM_N, raft_group=NEM_G, latency_dist="exponential", latency_mean_ms=5,  # noqa: E731
                            seed=0x4D41454C)
    oa, rows, ops = twins(NEM_N, NEM_G, nemesis_scenario, nem, oracle=oracle, **kw)
    assert len(rows) > 4
    sends = (oa["ev"]["event_id"] & RECV) == 0
    assert oa["stats"]["servers"]["send-count"] > oa["stats"]["servers"]["recv-count"]   # the cuts dropped replicates
    assert np.count_nonzero(sends & (oa["bd"]["type"] == REPLICATE)) > 20
    # the history, again, from one run on the engine
    s = mb.Sim(NEM_N, seed=0x4D41454C, **kw)
    from test_nemesis import DeviceNemesis
    hb, state = nemesis_scenario(s, lambda x: DeviceNemesis(x, **{k: v for k, v in nem.items() if k != "now0"}))
    s.close()
    h = np.frombuffer(hb, dtype=mb._lib.TXN_RW_HIST_DTYPE)
    assert np.count_nonzero(h["type"] == INVOKE) > 500
    assert check(h) == set()                                                # every op :ok, read committed holds
    # the finding: no read through a node returns a value written through its block partner ...
    node_of = {int(r["base"]): int(r["node"]) for r in h[h["type"] == INVOKE]}
    reads = [(int(r["node"]), v) for r in h[h["type"] == OK] for w, k, v in mops(r["ops"], r["base"], r["reads"])
             if not w and v]
    assert len(reads) > 100
    assert all(node_of[(v - 1) // 4 * 4 + 1] == nd for nd, v in reads)
    # ... and the partners' stores differ after the run
    for b in range(0, NEM_N, NEM_G):
        assert state[b][2] != state[b + 1][2]


# ------------------------------------------------------------------------------------------- scale (GPU)
SCALE_N, SCALE_C, SCALE_G = 4096, 16384, 2
SCALE = dict(ring_cap=64, max_window=64, server_ring_cap=64, server_max_window=32, journal_cap_log2=24,
             calendar_slots=64, max_endpoints=SCALE_N + SCALE_C + 8, raft_group=SCALE_G, gset_interval_ms=100)
SCALE_LIMIT = 3000
SCALE_STRETCHES = (1000, 2000, SCALE_LIMIT + 400)
SCALE_CLIENTS = dict(interval_ns=100 * MS, time_limit_ns=SCALE_LIMIT * MS, key_period_ns=500 * MS, key_count=4)


def scale_scenario(hist):
    def scenario(s, body):
        sink = s.add_endpoint("c99999", O.KIND_SIM_CLIENT)               # 32 init_ok a millisecond fit its ring
        s.schedule(ops_array([((i % 128) * MS, sink, i, "init", 1 + i, 0) for i in sorted(range(SCALE_N), key=lambda i: i % 128)]))
        s.run(130 * MS)
        s.add_txn_rw_clients(SCALE_C, **SCALE_CLIENTS)
        for t in SCALE_STRETCHES:
            s.run(t * MS)
            hist.append(s.txn_rw_history())
        return node_state(s, range(0, SCALE_N, 7))
    return scenario


@pytest.fixture(scope="module")
def scale_oracle():
    """the oracle twin's run of the scale scenario, once for the tests below"""
    o = RW.Sim(SCALE_N, raft_group=SCALE_G)
    ho = []
    state = scale_scenario(ho)(o, None)
    return o, state, np.concatenate(ho)


def scale_engine(**kw):
    import maelstrom_b200 as mb
    return mb.Sim(SCALE_N, workload="txn-rw-register", **dict(SCALE, **kw))


def check_scale(h):
    order = np.argsort(h["node"] // SCALE_G, kind="stable")
    hs = h[order]
    blocks, first = np.unique(hs["node"] // SCALE_G, return_index=True)
    assert len(blocks) == SCALE_N // SCALE_G
    for part in np.split(hs, first[1:]):                                   # every block, its records in history order
        assert check(part) == set()


@pytest.mark.gpu
def test_scale_2048_blocks_16384_clients(engine_backend, scale_oracle):
    if engine_backend != "cuda":
        pytest.skip("4096 txn-rw-register nodes: GPU only")
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
        pytest.skip("4096 txn-rw-register nodes: GPU only")
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
    """one block of 32: every node replicates to n0 in the same round, so n0 answers 31 replicates with 31 acks each"""
    start(s, 32)
    s.add_txn_rw_clients(32, interval_ns=10 * MS, time_limit_ns=250 * MS, key_period_ns=100 * MS, key_count=4)
    s.run(330 * MS)
    return s.txn_rw_history().tobytes(), node_state(s, (0, 1, 31))


@pytest.mark.gpu
def test_one_block_of_32_whose_lowest_node_sends_over_900_acks_a_step(engine_backend):
    if engine_backend != "cuda":
        pytest.skip("one block of 32: GPU only")
    import maelstrom_b200 as mb
    g = mb.Sim(32, workload="txn-rw-register", max_endpoints=80, ring_cap=2048, max_window=2048, server_ring_cap=2048,
               server_max_window=128, journal_cap_log2=22, gset_interval_ms=100)
    o = RW.Sim(32)
    (hg, sg), (ho, so) = both(g, o, wide_scenario)
    assert hg == ho and sg == so
    ev, bd = assert_same_journal(g, o)
    sends = ((ev["event_id"] & RECV) == 0) & (bd["type"] == REPLICATE_ACK) & (ev["src"] == 0)
    _, per_round = np.unique(ev["time_ns"][sends], return_counts=True)
    assert per_round.max() > 900
    g.close()
    o.close()
