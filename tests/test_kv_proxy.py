"""The lin-kv proxy (MS_W_KV_PROXY, DESIGN.md 2.14): demo/ruby/lin_kv_proxy.rb on node.rb, a node that forwards the
lin-kv workload's read / write / cas to a kv service and hands the service's reply back to the client.  Driven by the
closed-loop lin-kv clients (ms_add_kv_clients) over lin-kv, seq-kv and lww-kv.  Journal, stats, time, history and every
node's state must equal the proxy's oracle twin's (tests/native/kv_proxy_oracle.cpp); the proxy's rules are read back from the
journal; and the tutorial's lesson holds: linearizable over lin-kv, not over seq-kv or lww-kv."""
import ctypes as C
import json

import numpy as np
import pytest

import kv_proxy_oracle_lib as K
import oracle_lib as O
from scenarios import assert_same_journal, both, ops_array
from test_kv_clients import HIST_FIELDS, INVOKE, OK, TIMEOUT, check_every_key, linearizable
from test_round_shapes import windows

pytestmark = pytest.mark.usefixtures("engine_backend")
MS = 1_000_000
SERVICES = ("lin-kv", "seq-kv", "lww-kv")
RECV = np.uint64(1 << 63)
KV_TYPES = (O.T["read"], O.T["write"], O.T["cas"])


def proxy_pair(n, n_clients, service, g=3, **kw):
    """(engine, oracle twin) of n proxies over `service` with room for n_clients kv clients"""
    import maelstrom_b200 as mb
    args = dict(latency_dist="constant", latency_mean_ms=0, max_endpoints=n + n_clients + 8, ring_cap=256,
                max_window=256, server_ring_cap=64, server_max_window=64, raft_group=g, rpc_table=64, n_keys=64,
                journal_cap_log2=20, calendar_slots=64, calendar_cap=max(1024, 8 * n_clients))
    args.update(kw)
    shared = {k: args[k] for k in ("latency_dist", "latency_mean_ms", "p_loss", "raft_group", "rpc_table", "seed")
              if k in args}
    return (mb.Sim(n, workload="lin-kv-proxy", proxy_service=service, **args),
            K.Sim(n, proxy_service=service, **shared))


def start(s, n, service):
    """the service endpoint (index n), an init sink (n + 1), every node initialised in the first round"""
    svc = s.add_endpoint(service, O.KIND_SERVICE)
    sink = s.add_endpoint("c9999", O.KIND_SIM_CLIENT)
    s.schedule(ops_array([(0, sink, i, "init", 1 + i, 0) for i in range(n)]))
    s.run(5 * MS)
    return svc, sink


def clients_scenario(n, service, n_clients, until, jump=False, crash_at=None, **client_kw):
    kw = dict(interval_ns=10 * MS, time_limit_ns=until - 300 * MS, key_period_ns=150 * MS, keys_per_group=8)
    kw.update(client_kw)

    def scenario(s, body):
        if jump and hasattr(s, "idle_jump"):                # the oracle ticks: it is the reference for both runs
            s.idle_jump()
        start(s, n, service)
        host = s.add_endpoint("c9998", O.KIND_SIM_CLIENT) if crash_at is not None else None
        c0 = s.add_kv_clients(n_clients, **kw)
        if crash_at is not None:                          # a request type the node has no handler for: node 0 dies
            s.schedule(ops_array([(crash_at, host, 0, "echo", 1, 0)]))
        s.run(until)
        return c0
    return scenario


def run_pair(n, n_clients, service, scenario, **kw):
    """both sides of one scenario: everything observable must be equal; returns (engine, history, events, bodies)"""
    g, o = proxy_pair(n, n_clients, service, **kw)
    rg, ro = both(g, o, scenario)
    assert rg == ro
    hg, ho = g.history(), o.history()
    assert len(hg) == len(ho) > 0
    for f in HIST_FIELDS:
        assert np.array_equal(hg[f], ho[f]), f
    ev, bd = assert_same_journal(g, o)
    assert [g.proxy_state(i) for i in range(n)] == [o.proxy_state(i) for i in range(n)]
    o.close()
    return g, hg, ev, bd


# ------------------------------------------------------------------------------------------- the rules, from the journal
def check_proxy_rules(ev, bd, n, svc, rpc_table):
    """Every client request to a node is one RPC to the service, with that node's ids 1, 2, 3, ...; every reply of the
    service with a live closure is one answer to the client; a duplicate or stale reply is none.  Returns the number of
    service replies that found no live closure."""
    recv = (ev["event_id"] & RECV) != 0
    dropped = 0
    for e in range(n):
        reqs, rpcs, live, answers, sent_max = [], [], [], [], 0
        closures = {}
        for i in np.nonzero(((ev["dest"] == e) & recv) | ((ev["src"] == e) & ~recv))[0]:
            src, dest, b = int(ev["src"][i]), int(ev["dest"][i]), bd[i]
            if recv[i]:
                if src == svc and b["flags"] & O.F_REPLY:
                    k = int(b["in_reply_to"])
                    if k in closures and k > sent_max - rpc_table:   # the k-th RPC's slot still holds it
                        live.append((closures.pop(k), b))
                    else:
                        dropped += 1
                elif src > svc and b["type"] in KV_TYPES and not b["flags"] & O.F_REPLY:
                    reqs.append((src, b))
            elif dest == svc:
                rpcs.append(b)
                sent_max = int(b["msg_id"])
                closures[sent_max] = reqs[len(rpcs) - 1]
            elif b["type"] != O.T["init_ok"]:
                answers.append((dest, b))
        assert [int(b["msg_id"]) for b in rpcs] == list(range(1, len(rpcs) + 1))
        assert len(rpcs) == len(reqs)
        for (src, q), r in zip(reqs, rpcs):
            assert (r["type"], r["p0"], r["p1"]) == (q["type"], q["p0"], q["p1"])
            assert r["flags"] == O.F_MSG_ID | (q["flags"] & O.F_CREATE) and r["in_reply_to"] == 0
        assert len(answers) == len(live)
        for ((client, q), rep), (dest, a) in zip(live, answers):
            assert dest == client
            assert (a["type"], a["p0"], a["p1"]) == (rep["type"], rep["p0"], rep["p1"])
            assert a["flags"] == (int(rep["flags"]) & ~O.F_MSG_ID) and a["in_reply_to"] == q["msg_id"] and a["msg_id"] == 0
    return dropped


# ------------------------------------------------------------------------------------------- parity
CASES = [(svc, dist) for svc in SERVICES for dist in ("constant", "exponential")]


@pytest.mark.parametrize("service,dist", CASES)
def test_parity_with_the_kv_oracle_twin_jump_off_and_on(service, dist):
    n, n_clients = 6, 12
    net = dict(latency_dist="constant", latency_mean_ms=0) if dist == "constant" else \
        dict(latency_dist="exponential", latency_mean_ms=20, p_loss=0.1, rpc_table=2)
    # a short client timeout keeps the clients busy under loss; 2 closure slots make late replies stale
    client = dict(timeout_ns=150 * MS) if dist == "exponential" else {}
    runs = []
    for jump in (False, True):
        sc = clients_scenario(n, service, n_clients, 1600 * MS, jump, **client)
        g, h, ev, bd = run_pair(n, n_clients, service, sc, **net)
        runs.append((h, ev, bd, g.stats(), g.now, g.round, [g.proxy_state(i) for i in range(n)]))
        if jump:
            assert g.counters()["rounds"] < g.round                       # the jump skipped rounds
        g.close()
    (h0, ev0, bd0, *rest0), (h1, ev1, bd1, *rest1) = runs
    assert h0.tobytes() == h1.tobytes() and ev0.tobytes() == ev1.tobytes() and bd0.tobytes() == bd1.tobytes()
    assert rest0 == rest1
    inv = h0[h0["type"] == INVOKE]
    done = h0[h0["type"] != INVOKE]
    # the two groups work on the two clusters, on keys of their own: the proxies share the service's store
    group = (inv["client"] - (n + 2)) // 6
    keys = inv["value"] & 0xFFFF
    assert set(keys[group == 0].tolist()) == set(range(8)) and set(keys[group == 1].tolist()) == set(range(8, 16))
    assert len(inv) > 150 and np.count_nonzero(done["type"] == OK) > 30
    dropped = check_proxy_rules(ev0, bd0, n, n, net.get("rpc_table", 64))
    if dist == "exponential":
        assert dropped > 0 and np.count_nonzero(done["error"] == TIMEOUT) > 0   # stale replies were dropped
    else:
        assert dropped == 0 and len(done) == len(inv)


# ------------------------------------------------------------------------------------------- host-driven edges
def json_send(g, line):
    return g.L.ms_send_json(g.h, line.encode())


def json_recv(g, ep, timeout_ns=100 * MS):
    buf = C.create_string_buffer(1 << 16)
    rc = g.L.ms_recv_json(g.h, ep, timeout_ns, buf, len(buf))
    assert rc >= 0, g.L.ms_last_error(g.h).decode()
    return json.loads(buf.value.decode()) if rc == 1 else None


def host_scenario(s, body):
    """one host client against proxy n0 over lin-kv: msg_id-less requests, a second init, create_if_not_exists, errors
    passed on, replies without a live closure, then a request type without a handler"""
    s.add_endpoint("lin-kv", O.KIND_SERVICE)
    c = s.add_endpoint("c1", O.KIND_CLIENT)
    got = []

    def rpc(b, expect=True):
        s.send(c, 0, b)
        m = s.recv(c, 50 * MS)
        assert (m is not None) == expect
        if m is not None:
            got.append(tuple(int(m[k]) for k in ("src", "type", "flags", "msg_id", "in_reply_to", "p0", "p1")))
    rpc(body("init", msg_id=1))
    rpc(body("init", msg_id=2))                                            # a second init is answered too
    rpc(body("init"))                                                      # ... and one without msg_id: no in_reply_to
    rpc(body("write", p0=1, p1=7))                                         # no msg_id: write_ok without in_reply_to
    rpc(body("read", msg_id=3, p0=1))
    rpc(body("cas", msg_id=4, p0=2, p1=0 | 5 << 32))                       # missing key: error 20, passed on
    rpc(body("cas", msg_id=5, p0=2, p1=0 | 5 << 32, create=True))          # created
    rpc(body("cas", msg_id=6, p0=2, p1=4 | 6 << 32))                       # from mismatch: error 22
    rpc(body("read", msg_id=7, p0=2))
    rpc(body("read_ok", msg_id=8, in_reply_to=5, p1=9), expect=False)      # a reply its closure already took
    rpc(body("read_ok", in_reply_to=99, p1=9), expect=False)               # a reply nobody waits for
    state = s.proxy_state(0)
    rpc(body("echo", msg_id=9), expect=False)                              # no handler: the node dies
    rpc(body("read", msg_id=10, p0=2), expect=False)
    rpc(body("init", msg_id=11), expect=False)
    return got, state, s.proxy_state(0), s.proxy_state(1)


def test_host_driven_edges():
    g, o = proxy_pair(2, 0, "lin-kv", raft_group=0)
    import maelstrom_b200 as mb
    rg, ro = both(g, o, host_scenario)
    assert rg == ro
    got, before, after, other = rg
    R, M, C_ = O.F_REPLY, O.F_MSG_ID, O.F_CREATE
    T = O.T
    assert [x[1:5] for x in got] == [(T["init_ok"], R, 0, 1), (T["init_ok"], R, 0, 2), (T["init_ok"], 0, 0, 0),
                                     (T["write_ok"], 0, 0, 0), (T["read_ok"], R, 0, 3), (T["error"], R, 0, 4),
                                     (T["cas_ok"], R, 0, 5), (T["error"], R, 0, 6), (T["read_ok"], R, 0, 7)]
    assert [x[5] for x in got if x[1] == T["error"]] == [20, 22] and got[4][6] == 7 and got[8][6] == 5
    assert all(x[0] == 0 for x in got)
    assert before == {"crashed": 0, "next_msg_id": 6, "pending": 0}
    assert after == {"crashed": 1, "next_msg_id": 6, "pending": 0}
    assert other == {"crashed": 0, "next_msg_id": 0, "pending": 0}
    ev, bd = assert_same_journal(g, o)
    recv = (ev["event_id"] & RECV) != 0
    to_svc = ~recv & (ev["dest"] == 2)
    assert bd["flags"][to_svc].tolist() == [M, M, M, M | C_, M, M]           # create_if_not_exists passed through
    # the dead node still takes its mail off the network (:recv journaled) and never sends again
    crash = int(np.nonzero(recv & (ev["dest"] == 0) & (bd["type"] == T["echo"]))[0][0])
    assert np.count_nonzero((recv & (ev["dest"] == 0))[crash:]) == 3
    assert not np.any((~recv & (ev["src"] == 0))[crash:])
    g.close()
    o.close()
    # the same exchange through the JSON envelope
    with mb.Sim(2, workload="lin-kv-proxy") as s:
        s.add_endpoint("lin-kv", O.KIND_SERVICE)
        s.add_endpoint("c1", O.KIND_CLIENT)
        assert json_send(s, '{"src":"c1","dest":"n0","body":{"type":"cas","msg_id":1,"key":3,"from":1,"to":2,'
                            '"create_if_not_exists":true}}') >= 0
        assert json_recv(s, 3)["body"] == {"type": "cas_ok", "in_reply_to": 1}
        assert json_send(s, '{"src":"c1","dest":"n1","body":{"type":"read","msg_id":2,"key":3}}') >= 0
        m = json_recv(s, 3)
        assert (m["src"], m["dest"], m["body"]) == ("n1", "c1", {"type": "read_ok", "in_reply_to": 2, "value": 2})
        assert json_send(s, '{"src":"c1","dest":"n1","body":{"type":"write","key":4,"value":8}}') >= 0
        assert json_recv(s, 3)["body"] == {"type": "write_ok"}


def test_kv_clients_of_a_crashed_node_time_out():
    n, n_clients = 3, 12
    sc = clients_scenario(n, "lin-kv", n_clients, 2500 * MS, crash_at=500 * MS, time_limit_ns=2000 * MS)
    g, h, ev, bd = run_pair(n, n_clients, "lin-kv", sc)
    assert g.proxy_state(0)["crashed"] == 1 and g.proxy_state(1)["crashed"] == 0
    c0 = n + 3
    bound0 = (h["client"] - c0) % 3 == 0
    late = h[bound0 & (h["time_ns"] > 600 * MS) & (h["type"] != INVOKE)]
    assert len(late) > 0 and set(late["error"].tolist()) == {TIMEOUT}
    others = h[~bound0 & (h["time_ns"] > 600 * MS) & (h["type"] != INVOKE)]
    assert np.count_nonzero(others["type"] == OK) > 20
    recv = (ev["event_id"] & RECV) != 0
    crash = int(np.nonzero(recv & (ev["dest"] == 0) & (bd["type"] == O.T["echo"]))[0][0])
    assert np.count_nonzero((recv & (ev["dest"] == 0))[crash:]) > 5 and not np.any((~recv & (ev["src"] == 0))[crash:])
    g.close()


def test_missing_backing_service_and_refusals():
    import maelstrom_b200 as mb
    with mb.Sim(3, workload="lin-kv-proxy", proxy_service="seq-kv") as s:
        s.add_endpoint("lin-kv", O.KIND_SERVICE)                           # not the one the proxies forward to
        c = s.add_endpoint("c1", O.KIND_CLIENT)
        s.send(c, 1, mb.body("read", msg_id=1, p0=0))
        with pytest.raises(mb.SimError) as e:
            s.run(5 * MS)
        assert "Invalid dest" in str(e.value)
    for bad in (3, 7):                                                     # lin-tso, and no service at all
        with pytest.raises(mb.SimError) as e:
            mb.Sim(3, workload="lin-kv-proxy", proxy_service=bad)
        assert "reserved[3]" in str(e.value)
        with pytest.raises(RuntimeError):
            K.Sim(3, proxy_service=bad)
    with pytest.raises(mb.SimError) as e:
        mb.Sim(4, workload="lin-kv-proxy", n_shards=2, shard_id=0)
    assert "one GPU" in str(e.value)
    ok = dict(interval_ns=10 * MS, time_limit_ns=100 * MS, key_period_ns=50 * MS)
    with mb.Sim(6, workload="lin-kv-proxy", raft_group=3, n_keys=8, max_endpoints=64) as s:
        # not a multiple of 2g; two groups of 5 keys on two clusters, which Raft would take: the proxies share one store
        for kw in (dict(n_clients=9), dict(n_clients=12, keys_per_group=5)):
            with pytest.raises(mb.SimError) as e:
                s.add_kv_clients(**kw, **ok)
            assert e.value.code == -2 and "ms_add_kv_clients" in str(e.value)
        assert s.add_kv_clients(12, keys_per_group=4, **ok) == 6
        with pytest.raises(mb.SimError):                                   # once per simulation
            s.add_kv_clients(12, first_name=100, **ok)


# ------------------------------------------------------------------------------------------- the lesson
def lesson(service):
    n, n_clients = 3, 12
    sc = clients_scenario(n, service, n_clients, 2000 * MS, key_period_ns=100 * MS, keys_per_group=8,
                          interval_ns=20 * MS)
    g, h, _, _ = run_pair(n, n_clients, service, sc, seed=0x5EED)
    import maelstrom_b200 as mb
    per_key = mb.kv_history(h, *g.kv_groups)
    g.close()
    assert len(per_key) >= 8
    return g, h, per_key


def test_linearizable_over_lin_kv():
    g, h, per_key = lesson("lin-kv")
    check_every_key(g, h)


@pytest.mark.parametrize("service", ["seq-kv", "lww-kv"])
def test_not_linearizable_over_seq_kv_and_lww_kv(service):
    _, _, per_key = lesson(service)
    bad = [k for k, ops in per_key.items() if not linearizable(ops)]
    assert bad, "every register of the %s run is linearizable" % service


# ------------------------------------------------------------------------------------------- a class-3 service window
def test_service_window_above_2048():
    n, n_clients = 30, 2112                                                # 352 groups of 2g = 6; all invoke at once
    sc = clients_scenario(n, "lin-kv", n_clients, 60 * MS, interval_ns=20 * MS, time_limit_ns=40 * MS,
                          key_period_ns=1000 * MS, keys_per_group=1)
    g, h, ev, bd = run_pair(n, n_clients, "lin-kv", sc, ring_cap=4096, max_window=4096, server_ring_cap=256,
                            server_max_window=128, rpc_table=128, n_keys=512)
    svc_windows = [size for dest, size in windows(ev) if dest == n]
    assert max(svc_windows) > 2048
    assert check_proxy_rules(ev, bd, n, n, 128) == 0                       # a node has ~70 RPCs out at once
    g.close()


# ------------------------------------------------------------------------------------------- scale (GPU)
SCALE_N, SCALE_G = 4095, 5
SCALE = dict(raft_group=SCALE_G, ring_cap=8192, max_window=8192, server_ring_cap=64, server_max_window=32,
             rpc_table=64, n_keys=8192, journal_cap_log2=24, calendar_slots=64)
SCALE_STRETCHES = (1000, 2000, 3000)


def scale_scenario(service, hist):
    n, n_clients = SCALE_N, 2 * SCALE_N

    def scenario(s, body):
        start(s, n, service)
        s.add_kv_clients(n_clients, interval_ns=100 * MS, time_limit_ns=2700 * MS, key_period_ns=500 * MS,
                         keys_per_group=8)
        for t in SCALE_STRETCHES:
            s.run(t * MS)
            hist.append(s.history())
        return [s.proxy_state(i) for i in range(0, n, 97)]
    return scenario


@pytest.fixture(scope="module")
def scale_oracle():
    """the oracle twin's run of the lin-kv scale scenario, once for the tests below"""
    o = K.Sim(SCALE_N, proxy_service="lin-kv", raft_group=SCALE_G, rpc_table=64)
    ho = []
    states = scale_scenario("lin-kv", ho)(o, None)
    return o, states, np.concatenate(ho)


def scale_engine(service, **kw):
    import maelstrom_b200 as mb
    return mb.Sim(SCALE_N, workload="lin-kv-proxy", proxy_service=service,
                  max_endpoints=3 * SCALE_N + 8, **dict(SCALE, **kw))


def same_history(hg, ho):
    assert len(hg) == len(ho) > 4 * SCALE_N
    for f in HIST_FIELDS:
        assert np.array_equal(hg[f], ho[f]), f


@pytest.mark.gpu
def test_scale_4095_proxies_over_lin_kv(engine_backend, scale_oracle):
    if engine_backend != "cuda":
        pytest.skip("4095 proxies: GPU only")
    o, states, ho = scale_oracle
    g = scale_engine("lin-kv")
    hg = []
    assert scale_scenario("lin-kv", hg)(g, None) == states
    hg = np.concatenate(hg)
    same_history(hg, ho)
    ev, _ = assert_same_journal(g, o)
    assert max(size for dest, size in windows(ev) if dest == SCALE_N) > 4096
    done = hg[hg["type"] != INVOKE]
    assert np.count_nonzero(done["type"] == OK) > 4 * SCALE_N
    import maelstrom_b200 as mb
    per_key = mb.kv_history(hg[hg["client"] < SCALE_N + 2 + 10 * 40], *g.kv_groups)   # the first 40 groups
    assert len(per_key) >= 40
    for key, ops in per_key.items():
        assert linearizable(ops), key
    g.close()


@pytest.mark.gpu
def test_scale_streamed_with_the_history_drained_between_stretches(engine_backend, scale_oracle):
    if engine_backend != "cuda":
        pytest.skip("4095 proxies: GPU only")
    from test_stream_overlap import Streamer, compare
    o, states, ho = scale_oracle
    g = scale_engine("lin-kv", journal_level=1)
    s = Streamer(g, 8, 1 << 22, drain_between=True)
    hg = []
    assert scale_scenario("lin-kv", hg)(s, None) == states
    same_history(np.concatenate(hg), ho)
    compare(s.journal(), o, g)
    assert len(s.batches) > 3
    g.close()


@pytest.mark.gpu
def test_scale_4095_proxies_over_seq_kv(engine_backend):
    if engine_backend != "cuda":
        pytest.skip("4095 proxies: GPU only")
    o = K.Sim(SCALE_N, proxy_service="seq-kv", raft_group=SCALE_G, rpc_table=64)
    g = scale_engine("seq-kv")
    hg, ho = [], []
    rg, ro = scale_scenario("seq-kv", hg)(g, None), scale_scenario("seq-kv", ho)(o, None)
    assert rg == ro
    same_history(np.concatenate(hg), np.concatenate(ho))
    assert_same_journal(g, o)
    g.close()
    o.close()
