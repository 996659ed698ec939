"""The kafka workload (MS_W_KAFKA, DESIGN.md 2.15): demo/clojure/kafka_single_node.clj on the device, every node its own
append-only log per key, driven by the closed-loop kafka clients (ms_add_kafka_clients).  Journal, stats, time, the
kafka history, every node's logs and committed offsets must equal the oracle twin's (tests/native/kafka_oracle.cpp);
the node's rules are read back from host-driven exchanges; and the checker below (the kafka analyses this history
supports, restated) finds nothing with one server per client group and duplicate offsets with three: the demo is a
single-node log."""
import numpy as np
import pytest

import kafka_oracle_lib as K
import oracle_lib as O
from scenarios import assert_same_journal, both, ops_array

pytestmark = pytest.mark.usefixtures("engine_backend")
MS = 1_000_000
INVOKE, OK, FAIL, INFO = 0, 1, 2, 3
TIMEOUT = 0xFFFF
SEND, POLL, ASSIGN, CRASH = 10, 11, 12, 13                     # MS_HF_KAFKA_*
NO_KEY, NONE = 0xFFFF, 0xFFFFFFFF
KT = dict(send=70, send_ok=71, poll=72, poll_ok=73, commit_offsets=74, commit_offsets_ok=75,
          list_committed_offsets=76, list_committed_offsets_ok=77)
HIST_FIELDS = ("time_ns", "order", "client", "op", "type", "f", "error", "key", "a", "b")
RECV = np.uint64(1 << 63)


def kafka_pair(n, n_clients, g=1, keys=4, cap=4096, **kw):
    """(engine, oracle twin) of n kafka nodes with room for n_clients kafka clients"""
    import maelstrom_b200 as mb
    args = dict(latency_dist="constant", latency_mean_ms=0, max_endpoints=n + n_clients + 8, ring_cap=256,
                max_window=256, server_ring_cap=64, server_max_window=64, raft_group=g, journal_cap_log2=20,
                calendar_slots=64, calendar_cap=max(1024, 8 * n_clients))
    args.update(kw)
    shared = {k: args[k] for k in ("latency_dist", "latency_mean_ms", "p_loss", "raft_group", "seed") if k in args}
    return (mb.Sim(n, workload="kafka", kafka_keys=keys, kafka_log_cap=cap, **args),
            K.Sim(n, kafka_keys=keys, kafka_log_cap=cap, **shared))


def start(s, n):
    """an init sink (index n), every node initialised in the first round"""
    sink = s.add_endpoint("c99999", O.KIND_SIM_CLIENT)
    s.schedule(ops_array([(0, sink, i, "init", 1 + i, 0) for i in range(n)]))
    s.run(5 * MS)
    return sink


def clients_scenario(n, n_clients, until, jump=False, stretches=1, **client_kw):
    kw = dict(interval_ns=10 * MS, time_limit_ns=until - 300 * MS, assign_permille=100, crash_permille=20)
    kw.update(client_kw)

    def scenario(s, body):
        if jump and hasattr(s, "idle_jump"):                # the oracle ticks: it is the reference for both runs
            s.idle_jump()
        start(s, n)
        s.add_kafka_clients(n_clients, **kw)
        hist = []
        for k in range(1, stretches + 1):
            s.run(5 * MS + (until - 5 * MS) * k // stretches)
            hist.append(s.kafka_history())
        return np.concatenate(hist)
    return scenario


def node_state(s, n, keys):
    return ([s.kafka_log(i, k).tolist() for i in range(n) for k in range(keys)],
            [s.kafka_committed(i, k) for i in range(n) for k in range(keys)])


def same_history(hg, ho):
    assert len(hg) == len(ho) > 0
    for f in HIST_FIELDS:
        assert np.array_equal(hg[f], ho[f]), f


def run_pair(n, n_clients, scenario, keys=4, **kw):
    """both sides of one scenario: everything observable must be equal; returns (engine, history, events, bodies)"""
    g, o = kafka_pair(n, n_clients, keys=keys, **kw)
    hg, ho = both(g, o, scenario)
    same_history(hg, ho)
    ev, bd = assert_same_journal(g, o)
    assert node_state(g, n, keys) == node_state(o, n, keys)
    o.close()
    return g, hg, ev, bd


# ------------------------------------------------------------------------------------------- the checker
def check(h, logs, n_nodes, first, group):
    """The kafka analyses this history supports (jepsen.tests.kafka, restated).  `logs[node][key]` is ms_kafka_log;
    client c is on node (c - first) mod n_nodes, in group node / group.  A poll ok record names the messages
    logs[node][key][a:b].  Returns {anomaly: [cases]}."""
    bad = {k: [] for k in ("duplicate", "inconsistent", "lost", "nonmonotonic-send", "nonmonotonic-poll",
                           "skip-poll", "internal", "log")}
    node_of = lambda c: (int(c) - first) % n_nodes                 # noqa: E731
    at = {}                 # (group, key, offset) -> {msgs}
    where = {}              # (group, msg) -> {(key, offset)}
    polled = {}             # (group, key) -> {offsets observed}
    acked = []              # (group, key, offset, msg)
    ok = h[h["type"] == OK]

    def see(gr, key, off, msg):
        at.setdefault((gr, key, off), set()).add(msg)
        where.setdefault((gr, msg), set()).add((key, off))
    for r in ok:
        nd = node_of(r["client"])
        gr = nd // group
        if r["f"] == SEND:
            key, msg, off = int(r["key"][0]), int(r["a"][0]), int(r["b"][0])
            acked.append((gr, key, off, msg))
            see(gr, key, off, msg)
            log = logs[nd][key]
            if off >= len(log) or int(log[off]) != msg:
                bad["log"].append((int(r["client"]), key, off, msg))
        elif r["f"] == POLL:
            for s in range(2):
                key, a, b = int(r["key"][s]), int(r["a"][s]), int(r["b"][s])
                if key == NO_KEY:
                    continue
                if not a < b <= len(logs[nd][key]):
                    bad["internal"].append((int(r["client"]), key, a, b))
                    continue
                for off in range(a, b):
                    see(gr, key, off, int(logs[nd][key][off]))
                    polled.setdefault((gr, key), set()).add(off)
    for (gr, key, off), msgs in at.items():
        if len(msgs) > 1:
            bad["duplicate"].append((gr, key, off, sorted(msgs)))
    for (gr, msg), places in where.items():
        if len(places) > 1:
            bad["inconsistent"].append((gr, msg, sorted(places)))
    top = {}
    for (gr, key), offs in polled.items():
        top[(gr, key)] = max(offs)
    for gr, key, off, msg in acked:                               # an acked write below an observed offset, never read
        if off < top.get((gr, key), -1) and off not in polled[(gr, key)]:
            bad["lost"].append((gr, key, off, msg))
    exists = set((gr, key, off) for (gr, key, off) in at)
    # per client, reset at every assign and every :info (the client is reopened): offsets only go up, one by one
    last_send, last_poll = {}, {}
    for r in h[h["type"] != INVOKE]:
        c = int(r["client"])
        gr = node_of(c) // group
        if r["type"] == INFO or (r["f"] == ASSIGN and r["type"] == OK):
            last_send.pop(c, None)
            last_poll.pop(c, None)
            continue
        if r["type"] != OK:
            continue
        if r["f"] == SEND:
            key, off = int(r["key"][0]), int(r["b"][0])
            prev = last_send.setdefault(c, {}).get(key)
            if prev is not None and off <= prev:
                bad["nonmonotonic-send"].append((c, key, prev, off))
            last_send[c][key] = off
        elif r["f"] == POLL:
            for s in range(2):
                key, a, b = int(r["key"][s]), int(r["a"][s]), int(r["b"][s])
                if key == NO_KEY:
                    continue
                prev = last_poll.setdefault(c, {}).get(key)
                if prev is not None and a < prev:
                    bad["nonmonotonic-poll"].append((c, key, prev, a))
                elif prev is not None and any((gr, key, o) in exists for o in range(prev, a)):
                    bad["skip-poll"].append((c, key, prev, a))
                last_poll[c][key] = b
    return bad


def logs_of(s, n, keys):
    return [[s.kafka_log(i, k) for k in range(keys)] for i in range(n)]


# ------------------------------------------------------------------------------------------- parity
@pytest.mark.parametrize("dist", ["constant", "exponential"])
def test_parity_with_the_kafka_oracle_twin_jump_off_and_on(dist):
    n, n_clients = 6, 12
    net = dict(latency_dist="constant", latency_mean_ms=0) if dist == "constant" else \
        dict(latency_dist="exponential", latency_mean_ms=20, p_loss=0.1)
    client = dict(timeout_ns=150 * MS) if dist == "exponential" else {}   # timeouts under loss, stale replies
    runs = []
    for jump in (False, True):
        g, h, ev, bd = run_pair(n, n_clients, clients_scenario(n, n_clients, 1600 * MS, jump, stretches=2, **client),
                                **net)
        runs.append((h, ev, bd, g.stats(), g.now, g.round, node_state(g, n, 4)))
        if jump:
            assert g.counters()["rounds"] < g.round                       # the jump skipped rounds
        g.close()
    (h0, ev0, bd0, *rest0), (h1, ev1, bd1, *rest1) = runs
    assert h0.tobytes() == h1.tobytes() and ev0.tobytes() == ev1.tobytes() and bd0.tobytes() == bd1.tobytes()
    assert rest0 == rest1
    done = h0[h0["type"] != INVOKE]
    for f in (SEND, POLL, ASSIGN, CRASH):
        assert np.count_nonzero((done["f"] == f) & (done["type"] == (INFO if f == CRASH else OK))) > 3, f
    polls = done[(done["f"] == POLL) & (done["type"] == OK)]
    assert np.count_nonzero(polls["key"] != NO_KEY) > 10                  # polls that returned messages (and committed)
    assert any(c is not None for c in rest0[-1][1])
    if dist == "exponential":
        assert np.count_nonzero(done["error"] == TIMEOUT) > 0
    else:
        assert np.count_nonzero(done["error"] == TIMEOUT) == 0


# ------------------------------------------------------------------------------------------- the node, host-driven
def host_scenario(s, body):
    """one host client against node n0: sends, polls, commits, lists, an unknown type, a reply, msg_id-less requests"""
    c = s.add_endpoint("c1", O.KIND_CLIENT)
    got = []

    def rpc(b, expect=True):
        s.send(c, 0, b)
        m = s.recv(c, 50 * MS)
        assert (m is not None) == expect
        if m is not None:
            got.append(tuple(int(m[k]) for k in ("type", "flags", "in_reply_to", "p0", "p1")))

    def keys(k0, k1=NO_KEY):
        return k0 | k1 << 16
    rpc(body("init", msg_id=1))
    for i, (k, msg) in enumerate([(0, 7), (0, 8), (1, 9), (0, 10), (1, 11)]):
        rpc(body(KT["send"], msg_id=10 + i, p0=k, p1=msg))                     # offsets 0 1 0 2 1: dense per key
    rpc(body(KT["poll"], msg_id=20, p0=keys(0, 1), p1=1 | 0 << 32))           # [1, 3) of 0 and [0, 2) of 1
    rpc(body(KT["poll"], msg_id=21, p0=keys(0, 1), p1=3 | 1 << 32))           # past the end of 0: omitted
    rpc(body(KT["poll"], msg_id=22, p0=keys(2), p1=0))                        # an empty log: omitted
    rpc(body(KT["list_committed_offsets"], msg_id=23, p0=keys(0, 1)))         # nothing committed
    rpc(body(KT["commit_offsets"], msg_id=24, p0=keys(0, 1), p1=2 | 0 << 32))
    rpc(body(KT["commit_offsets"], msg_id=25, p0=keys(0), p1=1))              # never backwards
    rpc(body(KT["list_committed_offsets"], msg_id=26, p0=keys(0, 2)))         # 2 was never committed: omitted
    rpc(body(KT["list_committed_offsets"], msg_id=27, p0=keys(NO_KEY, 1)))
    rpc(body("echo", msg_id=28))                                              # unknown: error 10
    rpc(body(KT["send_ok"], msg_id=29, in_reply_to=3, p1=5), expect=False)    # a reply: ignored
    rpc(body(KT["send"], p0=3, p1=12))                                        # no msg_id: no in_reply_to
    rpc(body(KT["poll"], msg_id=30, p0=keys(3), p1=0))                        # the node goes on serving
    return got, node_state(s, 1, 4)


def test_node_rules_host_driven():
    g, o = kafka_pair(1, 0, keys=4)
    rg, ro = both(g, o, host_scenario)
    assert rg == ro
    got, (logs, committed) = rg
    R = O.F_REPLY
    err, init_ok = O.T["error"], O.T["init_ok"]
    assert got == [
        (init_ok, R, 1, 0, 0),
        (KT["send_ok"], R, 10, 0, 0), (KT["send_ok"], R, 11, 0, 1), (KT["send_ok"], R, 12, 0, 0),
        (KT["send_ok"], R, 13, 0, 2), (KT["send_ok"], R, 14, 0, 1),
        (KT["poll_ok"], R, 20, 0 | 1 << 16, 3 | 2 << 32),
        (KT["poll_ok"], R, 21, NO_KEY | 1 << 16, 0 | 2 << 32),
        (KT["poll_ok"], R, 22, NO_KEY | NO_KEY << 16, 0),
        (KT["list_committed_offsets_ok"], R, 23, NO_KEY | NO_KEY << 16, 0),
        (KT["commit_offsets_ok"], R, 24, 0, 0), (KT["commit_offsets_ok"], R, 25, 0, 0),
        (KT["list_committed_offsets_ok"], R, 26, 0 | NO_KEY << 16, 2),
        (KT["list_committed_offsets_ok"], R, 27, NO_KEY | 1 << 16, 0 << 32),
        (err, R, 28, 10, 0),
        (KT["send_ok"], 0, 0, 0, 0),
        (KT["poll_ok"], R, 30, 3 | NO_KEY << 16, 1)]
    assert logs == [[7, 8, 10], [9, 11], [], [12]] and committed == [2, 0, None, None]
    # the same exchange in the journal: one answer per request, none to the reply
    ev, bd = assert_same_journal(g, o)
    recv = (ev["event_id"] & RECV) != 0
    to_node = recv & (ev["dest"] == 0) & (ev["src"] == 1)
    from_node = ~recv & (ev["src"] == 0) & (ev["dest"] == 1)
    assert np.count_nonzero(to_node) == len(got) + 1 and np.count_nonzero(from_node) == len(got)
    g.close()
    o.close()


def test_refusals_and_latches():
    import maelstrom_b200 as mb
    with pytest.raises(mb.SimError) as e:
        mb.Sim(4, workload="kafka", n_shards=2, shard_id=0)
    assert "one GPU" in str(e.value)
    with pytest.raises(mb.SimError) as e:
        mb.Sim(2, workload="kafka", kafka_keys=65536)                    # keys are 16-bit, 0xFFFF is "no key"
    assert "reserved[2]" in str(e.value)
    ok = dict(interval_ns=10 * MS, time_limit_ns=100 * MS)
    with mb.Sim(3, workload="lin-kv") as s:                                # kafka clients on another workload
        with pytest.raises(mb.SimError) as e:
            s.add_kafka_clients(6, **ok)
        assert e.value.code == -2 and "MS_W_KAFKA" in str(e.value)
    with mb.Sim(3, workload="kafka", max_endpoints=64) as s:
        for kw in (dict(n_clients=4), dict(n_clients=6, assign_permille=600, crash_permille=401)):
            with pytest.raises(mb.SimError) as e:
                s.add_kafka_clients(**dict(ok, **kw))
            assert e.value.code == -2 and "ms_add_kafka_clients" in str(e.value)
        with pytest.raises(mb.SimError):                                   # the lin-kv clients are not for kafka
            s.add_kv_clients(6, interval_ns=MS, time_limit_ns=MS, key_period_ns=MS)
        assert s.add_kafka_clients(6, **ok) == 3
        with pytest.raises(mb.SimError):                                   # once per simulation
            s.add_kafka_clients(6, first_name=100, **ok)
        with pytest.raises(mb.SimError):
            s.raft_state(0)
        for bad in ((3, 0), (0, 16)):                                      # node, key out of range
            with pytest.raises(mb.SimError):
                s.kafka_log(*bad)
            with pytest.raises(mb.SimError):
                s.kafka_committed(*bad)
    with mb.Sim(2, workload="lin-kv") as s:
        with pytest.raises(mb.SimError):
            s.kafka_log(0, 0)
    # a full log, and a key out of range, latch a device error
    with mb.Sim(1, workload="kafka", kafka_keys=2, kafka_log_cap=2) as s:
        c = s.add_endpoint("c1", O.KIND_CLIENT)
        for i in range(2):
            s.send(c, 0, mb.body(KT["send"], msg_id=1 + i, p0=1, p1=i))
        s.run(3 * MS)
        assert s.kafka_log(0, 1).tolist() == [0, 1]
        s.send(c, 0, mb.body(KT["send"], msg_id=3, p0=1, p1=2))
        with pytest.raises(mb.SimError) as e:
            s.run(6 * MS)
        assert e.value.code == -3 and "kafka node's log of a key is full" in str(e.value)
    for req in (mb.body(KT["send"], msg_id=1, p0=2), mb.body(KT["poll"], msg_id=1, p0=NO_KEY << 16 | 5)):
        with mb.Sim(1, workload="kafka", kafka_keys=2) as s:
            c = s.add_endpoint("c1", O.KIND_CLIENT)
            s.send(c, 0, req)
            with pytest.raises(mb.SimError) as e:
                s.run(3 * MS)
            assert e.value.code == -3 and "value" in str(e.value)


# ------------------------------------------------------------------------------------------- the lesson
def lesson(g):
    n, n_clients, keys = 3, 12, 2
    sc = clients_scenario(n, n_clients, 2000 * MS, interval_ns=20 * MS, assign_permille=150, crash_permille=20)
    eng, h, _, _ = run_pair(n, n_clients, sc, keys=keys, g=g, seed=0x5EED)
    bad = check(h, logs_of(eng, n, keys), n, n + 1, g)
    eng.close()
    return h, bad


def test_one_node_per_group_is_a_correct_log():
    h, bad = lesson(1)
    assert {k: v for k, v in bad.items() if v} == {}
    ok = h[h["type"] == OK]
    assert np.count_nonzero(ok["f"] == SEND) > 100 and np.count_nonzero((ok["f"] == POLL) & (ok["key"][:, 0] != NO_KEY)) > 20


def test_three_nodes_per_group_give_duplicate_offsets():
    _, bad = lesson(3)
    assert bad["duplicate"] or bad["inconsistent"]
    assert not bad["log"] and not bad["internal"]                          # each node is still a correct log


# ------------------------------------------------------------------------------------------- scale (GPU)
SCALE_N, SCALE_C, SCALE_KEYS = 4096, 16384, 4
SCALE = dict(ring_cap=64, max_window=64, server_ring_cap=64, server_max_window=32, journal_cap_log2=24,
             calendar_slots=64, max_endpoints=SCALE_N + SCALE_C + 8)
SCALE_STRETCHES = (1000, 2000, 3000)


def scale_scenario(hist):
    def scenario(s, body):
        sink = s.add_endpoint("c99999", O.KIND_SIM_CLIENT)               # 32 init_ok a millisecond fit its ring
        s.schedule(ops_array([((i % 128) * MS, sink, i, "init", 1 + i, 0) for i in sorted(range(SCALE_N), key=lambda i: i % 128)]))
        s.run(130 * MS)
        s.add_kafka_clients(SCALE_C, interval_ns=100 * MS, time_limit_ns=2700 * MS, assign_permille=250,
                            crash_permille=100)
        for t in SCALE_STRETCHES:
            s.run(t * MS)
            hist.append(s.kafka_history())
        return node_state(s, SCALE_N, SCALE_KEYS)
    return scenario


@pytest.fixture(scope="module")
def scale_oracle():
    """the oracle twin's run of the scale scenario, once for the tests below"""
    o = K.Sim(SCALE_N, kafka_keys=SCALE_KEYS, kafka_log_cap=1024)
    ho = []
    state = scale_scenario(ho)(o, None)
    return o, state, np.concatenate(ho)


def scale_engine(**kw):
    import maelstrom_b200 as mb
    return mb.Sim(SCALE_N, workload="kafka", kafka_keys=SCALE_KEYS, kafka_log_cap=1024, **dict(SCALE, **kw))


@pytest.mark.gpu
def test_scale_4096_nodes_16384_clients(engine_backend, scale_oracle):
    if engine_backend != "cuda":
        pytest.skip("4096 kafka nodes: GPU only")
    o, state, ho = scale_oracle
    g = scale_engine()
    hg = []
    assert scale_scenario(hg)(g, None) == state
    hg = np.concatenate(hg)
    same_history(hg, ho)
    assert len(hg) > 8 * SCALE_C
    assert_same_journal(g, o)
    done = hg[hg["type"] != INVOKE]
    for f in (SEND, POLL, ASSIGN, CRASH):
        assert np.count_nonzero(done["f"] == f) > SCALE_C // 4, f
    bad = check(hg, logs_of(g, SCALE_N, SCALE_KEYS), SCALE_N, SCALE_N + 1, 1)
    assert {k: v[:5] for k, v in bad.items() if v} == {}
    g.close()


@pytest.mark.gpu
def test_scale_streamed_with_the_history_drained_between_stretches(engine_backend, scale_oracle):
    if engine_backend != "cuda":
        pytest.skip("4096 kafka nodes: GPU only")
    from test_stream_overlap import Streamer, compare
    o, state, ho = scale_oracle
    g = scale_engine(journal_level=1)
    s = Streamer(g, 8, 1 << 22, drain_between=True)
    hg = []
    assert scale_scenario(hg)(s, None) == state
    same_history(np.concatenate(hg), ho)
    compare(s.journal(), o, g)
    assert len(s.batches) > 3
    g.close()
