"""Closed-loop lin-kv clients on the device (ms_add_kv_clients, DESIGN.md 2.12): the worker of
workload/lin_kv.clj:40-85 driving the Raft nodes from inside the round kernel.  History, journal, stats and
node states must equal the oracle's; the history must obey the client rules and be what a register checker
needs: a brute-force linearizability search passes on every key and fails once a read is altered."""
import numpy as np
import pytest

import kv_oracle_lib as K
import oracle_lib as O
from scenarios import assert_same_journal, both, ops_array

pytestmark = pytest.mark.usefixtures("engine_backend")
INVOKE, OK, FAIL, INFO, TIMEOUT = 0, 1, 2, 3, 0xFFFF
READ, WRITE, CAS = 2, 3, 4
MS = 1_000_000
HIST_FIELDS = ("time_ns", "order", "client", "op", "type", "f", "error", "value")
G = 5                                   # servers per cluster
T0 = 4500 * MS                          # the first elections are over (2-4 s, raft.py:249-251)


def raft_pair(n, n_clients, **kw):
    args = dict(workload="lin-kv", latency_dist="constant", latency_mean_ms=1, max_endpoints=n + n_clients + 4,
                ring_cap=256, max_window=128, server_ring_cap=256, server_max_window=128, raft_group=G,
                rpc_table=256, n_keys=64, raft_log_cap=1024, journal_cap_log2=20, calendar_slots=64,
                calendar_cap=max(256, 8 * n))
    args.update(kw)
    import maelstrom_b200 as mb
    shared = {k: args[k] for k in ("latency_dist", "latency_mean_ms", "p_loss", "raft_group", "rpc_table") if k in args}
    # the oracle with the lin-kv clients' twin (tests/native/kv_oracle.cpp)
    return mb.Sim(n, **args), K.Sim(n, workload=O.W_RAFT, **shared)


def start(s, n):
    """init every node from one sink client, 32 per ms (its inbox takes that many init_ok), then let the clusters elect"""
    c = s.add_endpoint("c9999", O.KIND_SIM_CLIENT)
    s.schedule(ops_array([(i // 32 * MS, c, i, "init", 1 + i, 0) for i in range(n)]))
    s.run(T0)
    return c


def leaders(s, n):
    return [i for i in range(n) if s.raft_state(i)["state"] == 3]


def run_pair(n, n_clients, scenario, **kw):
    g, o = raft_pair(n, n_clients, **kw)
    rg, ro = both(g, o, scenario)
    assert rg == ro
    hg, ho = g.history(), o.history()
    assert len(hg) == len(ho) > 0
    for f in HIST_FIELDS:
        assert np.array_equal(hg[f], ho[f]), f
    ev, bd = assert_same_journal(g, o)
    assert [g.raft_state(i) for i in range(n)] == [o.raft_state(i) for i in range(n)]
    return g, hg, ev, bd


def healthy(n=15, n_clients=30, limit=T0 + 700 * MS, until=T0 + 1900 * MS, **client_kw):
    kw = dict(interval_ns=20 * MS, time_limit_ns=limit, key_period_ns=200 * MS, keys_per_group=8)
    kw.update(client_kw)

    def scenario(s, body):
        start(s, n)
        c0 = s.add_kv_clients(n_clients, **kw)
        assert c0 == n + 1
        s.run(until)
        return c0
    return scenario


def partitioned(n=15, n_clients=30):
    # every leader is isolated from its cluster for 5 s, then the partition heals (the shape of
    # tests/golden/raft_reference_trace_partition.json); a short timeout makes slow commits time out too
    def scenario(s, body):
        start(s, n)
        s.add_kv_clients(n_clients, interval_ns=40 * MS, time_limit_ns=T0 + 8000 * MS, key_period_ns=500 * MS,
                         keys_per_group=32, timeout_ns=120 * MS)
        s.run(T0 + 500 * MS)
        lead = leaders(s, n)
        s.partition([1 + i if i in lead else 0 for i in range(n)])       # clients (index >= n) are never cut
        s.run(T0 + 5500 * MS)
        s.heal()
        s.run(T0 + 9500 * MS)
        return lead
    return scenario


# ------------------------------------------------------------------------------------------- what the history says
def client_replies(ev, bd, n):
    """:recv events of replies at the generator's clients (endpoints above the init sink n)"""
    recv = (ev["event_id"] >> np.uint64(63)) == 1
    return recv & (ev["dest"] > n) & ((bd["flags"] & O.F_REPLY) != 0)


def check_client_rules(h, n, n_clients, limit, period, kpg, value_range=5, n_clusters=None):
    c0 = n + 1
    n_clusters = n_clusters or n // G
    for c in np.unique(h["client"]):
        mine = h[h["client"] == c]
        k = int(c) - c0
        assert 0 <= k < n_clients
        reader = k % (2 * G) < G
        base = (k // (2 * G)) // n_clusters * kpg
        open_op = None
        for r in mine:
            v = int(r["value"])
            key, a, b = v & 0xFFFF, (v >> 16) & 0xFF, v >> 24
            if r["type"] == INVOKE:
                assert open_op is None, "client %d invoked op %d while op %d was outstanding" % (c, r["op"], open_op[0])
                open_op = (int(r["op"]), int(r["f"]), v)
                assert r["time_ns"] < limit
                assert (r["f"] == READ) == reader and r["f"] in (READ, WRITE, CAS)
                assert key == base + (int(r["time_ns"]) // period) % kpg
                assert a < value_range and b < value_range
                assert (a, b) == (0, 0) if r["f"] == READ else b == 0 or r["f"] == CAS
            else:
                assert open_op is not None and open_op[:2] == (int(r["op"]), int(r["f"]))
                if r["f"] == READ and r["type"] == OK:
                    assert v & 0xFFFF == open_op[2] and a < value_range
                else:
                    assert v == open_op[2]
                open_op = None
        ops = mine[mine["type"] == INVOKE]["op"]
        assert ops.tolist() == list(range(1, len(ops) + 1))


def linearizable(ops):
    """Wing-Gong search over one key's history (mb.kv_history): a register with read / write / cas, initially
    missing.  :fail ops never happened, :info ops may take effect at any time after their invocation or never."""
    calls, open_by = [], {}
    for i, op in enumerate(ops):
        if op["type"] == "invoke":
            open_by[op["process"]] = len(calls)
            calls.append(dict(f=op["f"], value=op["value"][1], inv=i, ret=None, type="info"))
        else:
            c = calls[open_by.pop(op["process"])]
            c["type"], c["ret"] = op["type"], i
            if op["f"] == "read":
                c["value"] = op["value"][1]
    calls = [c for c in calls if c["type"] != "fail" and not (c["type"] == "info" and c["f"] == "read")]
    inf = len(ops) + 1
    for c in calls:
        if c["type"] == "info":
            c["ret"] = inf
    must = sum(1 << i for i, c in enumerate(calls) if c["type"] == "ok")
    seen, stack = set(), [(0, None)]
    while stack:
        done, state = stack.pop()
        if done & must == must:
            return True
        todo = [i for i in range(len(calls)) if not done >> i & 1]
        first_ret = min(calls[i]["ret"] for i in todo)
        for i in todo:
            c = calls[i]
            if c["inv"] > first_ret:
                continue
            if c["f"] == "read":
                if state != c["value"]:
                    continue
                nxt = state
            elif c["f"] == "write":
                nxt = c["value"]
            else:
                if c["type"] == "ok" and state != c["value"][0]:
                    continue
                nxt = c["value"][1] if state == c["value"][0] else state     # an :info cas may have failed
            node = (done | 1 << i, nxt)
            if node not in seen:
                seen.add(node)
                stack.append(node)
    return False


def check_every_key(g, h, min_ok_reads=1):
    import maelstrom_b200 as mb
    per_key = mb.kv_history(h, *g.kv_groups)
    assert len(per_key) > 3
    for key, ops in per_key.items():
        assert linearizable(ops), "register %s is not linearizable" % (key,)
    # negative control: one :ok read altered to a value nobody ever wrote
    altered = 0
    for key, ops in per_key.items():
        reads = [i for i, op in enumerate(ops) if op["f"] == "read" and op["type"] == "ok"]
        if not reads:
            continue
        bad = [dict(op) for op in ops]
        bad[reads[len(reads) // 2]]["value"] = (key[1], 200)
        assert not linearizable(bad), "register %s: an altered read went unnoticed" % (key,)
        altered += 1
    assert altered >= min_ok_reads
    return per_key


# ------------------------------------------------------------------------------------------- parity
@pytest.mark.parametrize("dist,mean,loss", [("constant", 1, 0.0), ("exponential", 3, 0.0), ("constant", 1, 0.1)])
def test_parity_rules_and_linearizability(dist, mean, loss):
    n, n_clients = 15, 30
    limit = T0 + 700 * MS
    g, h, ev, bd = run_pair(n, n_clients, healthy(n, n_clients, limit), latency_dist=dist, latency_mean_ms=mean, p_loss=loss)
    check_client_rules(h, n, n_clients, limit, 200 * MS, 8)
    inv = h[h["type"] == INVOKE]
    assert len(inv) > (50 if loss else 150) and set(inv["f"].tolist()) == {READ, WRITE, CAS}
    assert len(set(h["client"].tolist())) == n_clients
    done = h[h["type"] != INVOKE]
    assert np.count_nonzero(done["type"] == OK) > (10 if loss else 60)
    # default timeout = max(10 x latency mean, 1000) ms (lin_kv.clj:54); every op ended one way or the other
    assert len(done) == len(inv)
    to = done[done["error"] == TIMEOUT]
    if loss:
        assert len(to) > 0
    for r in to:
        mine = inv[(inv["client"] == r["client"]) & (inv["op"] == r["op"])]
        assert int(r["time_ns"]) - int(mine[0]["time_ns"]) == max(10 * mean, 1000) * MS
    # no client hears from a server outside its cluster: the clusters are independent
    rep = client_replies(ev, bd, n)
    k = ev["dest"][rep].astype(np.int64) - (n + 1)
    assert np.array_equal(ev["src"][rep] // G, (k // (2 * G)) % (n // G))
    check_every_key(g, h)
    g.close()


def test_partitioned_leaders_timeouts_errors_proxies_and_stale_replies():
    n, n_clients = 15, 30
    g, h, ev, bd = run_pair(n, n_clients, partitioned(n, n_clients), raft_log_cap=4096)
    check_client_rules(h, n, n_clients, T0 + 8000 * MS, 500 * MS, 32)
    done = h[h["type"] != INVOKE]
    to = done[done["error"] == TIMEOUT]
    assert len(to) > 0
    assert set(to[to["f"] == READ]["type"].tolist()) <= {FAIL} and set(to[to["f"] != READ]["type"].tolist()) == {INFO}
    assert np.count_nonzero(done["error"] == 11) > 0                      # "not a leader": :fail
    assert set(done[(done["error"] > 0) & (done["error"] != TIMEOUT)]["type"].tolist()) == {FAIL}
    assert g.counters()["partition_drops"] > 0
    # proxied replies: the leader answers what a follower was asked
    rep = client_replies(ev, bd, n)
    k = ev["dest"][rep].astype(np.int64) - (n + 1)
    bound = ((k // (2 * G)) % (n // G)) * G + k % G
    assert np.count_nonzero(ev["src"][rep] != bound) > 0
    assert np.array_equal(ev["src"][rep] // G, bound // G)
    # stale replies: more replies arrived than ops were completed by one
    assert np.count_nonzero(rep) > np.count_nonzero(done["error"] != TIMEOUT)
    check_every_key(g, h)
    g.close()


def test_groups_share_a_cluster_on_disjoint_keys_and_values_follow_the_range():
    # 2 groups on the one whole cluster of 7 servers in clusters of 5 (the last 2 servers are a cluster without clients)
    n, n_clients = 7, 20
    limit = T0 + 400 * MS
    sc = healthy(n, n_clients, limit, T0 + 1600 * MS, keys_per_group=3, key_period_ns=100 * MS, value_range=3)
    g, h, ev, bd = run_pair(n, n_clients, sc, n_keys=6)
    check_client_rules(h, n, n_clients, limit, 100 * MS, 3, value_range=3, n_clusters=1)
    keys = h["value"] & 0xFFFF
    first = h["client"] < n + 1 + 10
    assert set(keys[first].tolist()) <= {0, 1, 2} and set(keys[~first].tolist()) <= {3, 4, 5}
    assert len(set(keys.tolist())) == 6
    assert int(ev["src"][client_replies(ev, bd, n)].max()) < G
    g.close()


# ------------------------------------------------------------------------------------------- errors
def test_bad_configurations_are_refused(engine_backend):
    import maelstrom_b200 as mb
    ok = dict(interval_ns=10 * MS, time_limit_ns=100 * MS, key_period_ns=50 * MS)

    def refused(s, *a, **kw):
        with pytest.raises(mb.SimError) as e:
            s.add_kv_clients(*a, **kw)
        assert e.value.code == -2 and "ms_add_kv_clients" in str(e.value)

    with mb.Sim(9, workload="broadcast", max_endpoints=64) as s:
        refused(s, 18, **ok)                                              # not the Raft workload
        s.add_gen_clients(4, interval_ns=MS, time_limit_ns=10 * MS)
        refused(s, 18, **ok)                                              # ... nor after ms_add_gen_clients
    with mb.Sim(10, workload="lin-kv", raft_group=5, n_keys=8, max_endpoints=64) as s:
        refused(s, 15, **ok)                                              # not a multiple of 2g
        refused(s, 20, keys_per_group=9, **ok)                            # key range beyond ms_config.reserved[2]
        refused(s, 40, keys_per_group=5, **ok)                            # two groups per cluster: 10 keys
        refused(s, 20, keys_per_group=0, **ok)
        refused(s, 20, value_range=257, **ok)
        refused(s, 20, interval_ns=10 * MS, time_limit_ns=100 * MS, key_period_ns=0)
        assert s.add_kv_clients(20, keys_per_group=8, **ok) == 10
        refused(s, 20, first_name=100, **ok)                              # once per simulation
        with pytest.raises(mb.SimError):
            s.add_gen_clients(4, interval_ns=MS, time_limit_ns=10 * MS)
    with mb.Sim(10, workload="lin-kv", max_endpoints=64) as s:            # one cluster of all servers: 2g = 20
        refused(s, 10, **ok)
        assert s.add_kv_clients(20, **ok) == 10
    with mb.Sim(10, workload="lin-kv", raft_group=5, max_endpoints=64, n_shards=2, shard_id=0) as s:
        refused(s, 20, **ok)                                              # single GPU only
    o = K.Sim(10, workload=O.W_RAFT, raft_group=5)
    with pytest.raises(RuntimeError):
        o.add_kv_clients(15, **ok)


def test_history_ring_overflow_is_latched(engine_backend):
    # nodes that were never initialised answer "not a leader" at once: two records per op, never drained
    import maelstrom_b200 as mb
    with mb.Sim(10, workload="lin-kv", raft_group=5, max_endpoints=64, journal_level=0) as s:
        s.add_kv_clients(40, interval_ns=MS // 2, time_limit_ns=10_000 * MS, key_period_ns=100 * MS)
        with pytest.raises(mb.SimError) as e:
            s.run(3000 * MS)
        assert "history ring" in str(e.value)


# ------------------------------------------------------------------------------------------- scale (GPU)
def nemesis_scenario(n, n_clients, stretches, hist):
    # the partition nemesis of bench.py's raft config, one cycle: random halves for the first stretch, then healed.
    # (From a second cycle on some cluster of 819 reaches the reference's runaway regime, a leader that replicates
    # in every loop iteration, DESIGN.md 2.3, and its append_entries payloads outrun the payload heap.)  About one op
    # per client and second: reads are log entries too, a follower that lags is sent the whole suffix again and
    # again (DESIGN.md 2.8), and the payload heap has 64 vectors per node for what one round sends.
    def scenario(s, body):
        start(s, n)
        s.add_kv_clients(n_clients, interval_ns=1000 * MS, time_limit_ns=T0 + 2800 * MS, key_period_ns=500 * MS,
                         keys_per_group=8)
        rng = np.random.default_rng(5)
        for k, t in enumerate(stretches):
            if k == 0:
                s.partition(rng.integers(0, 2, size=n).astype(np.uint32))
            elif k == 1:
                s.heal()
            s.run(T0 + t * MS)
            h = s.history()
            hist.append(h)
        return [s.raft_state(i) for i in range(0, n, 97)]
    return scenario


SCALE = dict(latency_dist="constant", latency_mean_ms=0, server_ring_cap=64, server_max_window=32, rpc_table=64,
             n_keys=16, raft_log_cap=512, journal_cap_log2=24, ring_cap=64, max_window=32)


STRETCHES = (1000, 2000, 3000, 4000)


@pytest.fixture(scope="module")
def scale_oracle():
    """the oracle's run of the scale scenario, once for both tests: (simulation, node states, history)"""
    n = 4095                                                            # 819 clusters of 5
    _, o = raft_pair(n, 2 * n, **SCALE)
    ho = []
    states = nemesis_scenario(n, 2 * n, STRETCHES, ho)(o, None)
    return o, states, np.concatenate(ho)


@pytest.mark.gpu
def test_scale_4096_nodes_under_the_partition_nemesis(engine_backend, scale_oracle):
    if engine_backend != "cuda":
        pytest.skip("4096 nodes: GPU only")
    n = 4095
    n_clients = 2 * n
    o, states, ho = scale_oracle
    g, o_unused = raft_pair(n, n_clients, **SCALE)
    o_unused.close()
    hg = []
    assert nemesis_scenario(n, n_clients, STRETCHES, hg)(g, None) == states
    hg = np.concatenate(hg)
    assert len(hg) == len(ho) > 4 * n
    for f in HIST_FIELDS:
        assert np.array_equal(hg[f], ho[f]), f
    assert_same_journal(g, o)
    done = hg[hg["type"] != INVOKE]
    assert np.count_nonzero(done["type"] == OK) > n and np.count_nonzero(done["error"] == TIMEOUT) > 0
    check_client_rules(hg[hg["client"] < n + 1 + 200], n, n_clients, T0 + 2800 * MS, 500 * MS, 8)
    import maelstrom_b200 as mb
    per_key = mb.kv_history(hg[hg["client"] < n + 1 + 10 * 40], *g.kv_groups)   # the first 40 clusters
    assert len(per_key) > 40
    for key, ops in per_key.items():
        assert linearizable(ops), key
    g.close()


@pytest.mark.gpu
def test_scale_streamed_journal_with_the_history_drained_between_stretches(engine_backend, scale_oracle):
    if engine_backend != "cuda":
        pytest.skip("4096 nodes: GPU only")
    from test_stream_overlap import Streamer, compare
    n = 4095
    n_clients = 2 * n
    o, states, ho = scale_oracle
    g, o_unused = raft_pair(n, n_clients, journal_level=1, **SCALE)
    o_unused.close()
    s = Streamer(g, 8, 1 << 22, drain_between=True)
    hg = []
    assert nemesis_scenario(n, n_clients, STRETCHES, hg)(s, None) == states
    hg = np.concatenate(hg)
    assert len(hg) == len(ho) > 4 * n
    for f in HIST_FIELDS:
        assert np.array_equal(hg[f], ho[f]), f
    compare(s.journal(), o, g)
    assert len(s.batches) > 4
    g.close()
