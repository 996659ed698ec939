"""Idle-time jump (ms_set_idle_jump, DESIGN.md 2.3): with the mode on, ms_run, ms_run_streamed and the waiting
loop of ms_recv move virtual time and the round counter straight to the next tick at which an endpoint acts.  Every
output must be byte-identical to the same calls made without the mode: each case runs the same scenario twice on
the engine (ticking, jumping) and, where the oracle has the node program, once on the oracle, and compares
journal, bodies, history, statistics, node states, ms_now and ms_round.  A floor on the share of rounds jumped keeps
a mode that never jumps from passing.  [emul] = the kernel sources on the CPU SIMT emulator, [cuda] = an H100."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import kv_oracle_lib as K
import oracle_lib as O
from scenarios import ops_array

pytestmark = pytest.mark.usefixtures("engine_backend")
MS = 1_000_000
HIST_FIELDS = ("time_ns", "order", "client", "op", "type", "f", "error", "value")


def outputs(s, n_nodes, workload):
    ev, bd = s.drain()
    out = {"ev": ev, "bd": bd, "stats": s.stats(), "now": s.now, "round": s.round,
           "client_replies": s.client_replies(), "undeliverable": s.undeliverable()}
    if workload in ("broadcast", "g-set"):
        out["sets"] = [s.node_set(k).tolist() for k in range(n_nodes)]
    if workload == "lin-kv":
        out["raft"] = [s.raft_state(k) for k in range(n_nodes)]
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
    if "hist" in a and "hist" in b:
        assert len(a["hist"]) == len(b["hist"]), what
        for f in HIST_FIELDS:
            assert np.array_equal(a["hist"][f], b["hist"][f]), (what, f)


def engine(n, **kw):
    import maelstrom_b200 as mb
    return mb.Sim(n, **kw)


def run_twins(n, scenario, min_jumped, oracle=None, origin=0, jump_first=False, **kw):
    """The scenario on a ticking and a jumping engine (and an oracle, if given): returns (ticking, jumping) outputs
    and the scenario's results.  min_jumped: the least share of rounds the jumping engine must skip."""
    import maelstrom_b200 as mb
    workload = kw.get("workload", "broadcast")
    res, outs = [], []
    for jump in ((True, False) if jump_first else (False, True)):
        s = engine(n, **kw)
        if origin:
            s.set_origin(round=origin)
        if jump:
            assert s.idle_jump() == 0
        r = scenario(s, mb.body)
        o = outputs(s, n, workload)
        o["hist"] = s.history()
        o["rounds_run"] = s.counters()["rounds"]
        res.append(r)
        outs.append(o)
        s.close()
    if jump_first:
        res.reverse()
        outs.reverse()
    tick, jmp = outs
    assert res[0] == res[1]
    rounds_t, rounds_j = tick.pop("rounds_run"), jmp.pop("rounds_run")
    assert_same(tick, jmp, "jumping engine vs ticking engine")
    total = tick["round"] - origin
    assert rounds_t == total                                  # the ticking engine runs every round
    assert (total - rounds_j) >= min_jumped * total, (total, rounds_j)
    if oracle is not None:
        o = oracle()
        ro = scenario(o, O.body)
        assert ro == res[1]
        ev, bd = o.journal()
        oo = {"ev": ev, "bd": bd, "stats": o.stats(), "now": o.now, "round": o.round,
              "client_replies": o.client_replies(), "undeliverable": o.undeliverable()}
        if workload in ("broadcast", "g-set"):
            oo["sets"] = [o.node_set(k).tolist() for k in range(n)]
        if workload == "lin-kv":
            oo["raft"] = [o.raft_state(k) for k in range(n)]
        if hasattr(o, "history"):
            oo["hist"] = o.history()
        assert_same(jmp, oo, "jumping engine vs oracle")
        o.close()
    return tick, jmp, res[1]


def oracle_of(n, **kw):
    workload = kw["workload"]
    code = {"echo": O.W_ECHO, "broadcast": O.W_BROADCAST, "g-set": O.W_GSET, "txn-list-append": O.W_TXN,
            "txn-list-append-tree": O.W_TXN_TREE}[workload]
    # what scenarios.make_pair hands the oracle: everything but the engine's sizing
    keep = {k: v for k, v in kw.items() if k != "workload" and k not in (
        "max_endpoints", "ring_cap", "max_window", "journal_cap_log2", "journal_level", "calendar_slots", "calendar_cap",
        "mailbox_cap", "inject_cap", "threads_per_node", "n_keys", "raft_log_cap", "history_rounds", "server_ring_cap",
        "server_max_window")}
    return lambda: O.Sim(n, workload=code, **keep)


# ----------------------------------------------------------------------------------------------- every family
def sparse_echo(s, body):
    c = s.add_endpoint("c0", O.KIND_SIM_CLIENT)
    s.schedule(ops_array([(t * MS, c, i % 3, "echo", i + 1, i) for i, t in enumerate([0, 37, 38, 500, 2300, 2300])]))
    s.run(1200 * MS)
    s.schedule(ops_array([(3100 * MS, c, 1, "echo", 10, 10)]))
    s.run(4000 * MS)
    return s.client_replies()


def test_echo_sparse_scheduled_ops():
    kw = dict(workload="echo", max_endpoints=8, ring_cap=64, max_window=64)
    tick, jmp, replies = run_twins(3, sparse_echo, 0.95, oracle=oracle_of(3, **kw), **kw)
    assert replies == 7 and jmp["now"] == 4000 * MS


def broadcast_clients(s, body):
    s.add_gen_clients(4, interval_ns=250 * MS, time_limit_ns=2500 * MS, read_permille=400, timeout_ns=600 * MS,
                      quiet_ns=400 * MS, first_name=0)
    s.run(1500 * MS)
    s.flaky()                                         # loss 0.5 for a while: timeouts
    s.run(2000 * MS)
    s.set_loss(0.05)
    s.run(4500 * MS)
    return s.now


def test_broadcast_gen_clients_loss_exponential_latency():
    kw = dict(workload="broadcast", topology="grid", n_values=1 << 10, latency_dist="exponential", latency_mean_ms=100,
              p_loss=0.05, max_endpoints=16, ring_cap=256, max_window=128, calendar_slots=256, calendar_cap=4096, seed=11)
    tick, jmp, _ = run_twins(9, broadcast_clients, 0.2, oracle=oracle_of(9, **kw), **kw)
    h = jmp["hist"]
    assert len(h) > 20 and (h["type"] == 3).any()     # some ops timed out (:info)


def gset_periodic(s, body):
    c = s.add_endpoint("c0", O.KIND_SIM_CLIENT)
    s.schedule(ops_array([(0, c, i, "init", i + 1, 0) for i in range(4)] +
                         [(t * MS, c, t % 4, "add", 100 + t, v) for t, v in ((1, 1), (700, 7), (5200, 52), (9000, 9))]))
    s.run(16_000 * MS)
    return [s.node_set(k).tolist() for k in range(4)]


def test_gset_periodic_task():
    kw = dict(workload="g-set", latency_dist="constant", latency_mean_ms=20, n_values=64, max_endpoints=8,
              ring_cap=64, max_window=64, calendar_slots=64, calendar_cap=1024)
    tick, jmp, sets = run_twins(4, gset_periodic, 0.95, oracle=oracle_of(4, **kw), **kw)
    assert all(v == [1, 7, 9, 52] for v in sets)


def kv_partitioned(s, body):
    n = 5
    c = s.add_endpoint("c9999", O.KIND_SIM_CLIENT)
    s.schedule(ops_array([(0, c, i, "init", 1 + i, 0) for i in range(n)]))
    s.run(4500 * MS)
    s.add_kv_clients(10, interval_ns=300 * MS, time_limit_ns=12_000 * MS, key_period_ns=2000 * MS, keys_per_group=4,
                     timeout_ns=400 * MS)
    s.run(5000 * MS)
    lead = [i for i in range(n) if s.raft_state(i)["state"] == 3]
    s.partition([1 + i if i in lead else 0 for i in range(n)])
    s.run(10_000 * MS)
    s.heal()
    s.run(14_000 * MS)
    return lead


def test_raft_kv_clients_leaders_isolated():
    kw = dict(workload="lin-kv", latency_dist="constant", latency_mean_ms=1, max_endpoints=16, ring_cap=256,
              max_window=128, server_ring_cap=256, server_max_window=128, raft_group=5, rpc_table=256, n_keys=64,
              raft_log_cap=1024, journal_cap_log2=20, calendar_slots=64, calendar_cap=1024)
    oracle = lambda: K.Sim(5, workload=O.W_RAFT, latency_dist="constant", latency_mean_ms=1, raft_group=5, rpc_table=256)
    tick, jmp, lead = run_twins(5, kv_partitioned, 0.3, oracle=oracle, **kw)
    h = jmp["hist"]
    assert lead and (h["error"] == 11).any()          # requests to the isolated leader time out / fail


def single_key_txn(s, body):
    s.add_endpoint("lin-kv", O.KIND_SERVICE)
    cs = [s.add_endpoint("c%d" % i) for i in range(3)]
    for i in range(3):
        s.send(cs[i], i, body("init", msg_id=1))
    out = []
    for i in range(3):
        r = s.recv(cs[i], 1000 * MS)
        out.append(int(r["type"]))
    s.run(700 * MS)
    for k in range(3):
        s.send(cs[k], k, body("txn", msg_id=2 + k, p1=200 + k, appends=True))
        r = s.recv(cs[k], 300 * MS)
        out.append(None if r is None else (int(r["type"]), int(r["p0"]), int(r["p1"])))
        s.run(s.now + 900 * MS)
    return out


def test_single_key_txn_over_lin_kv():
    kw = dict(workload="txn-list-append", max_endpoints=16, latency_dist="constant", latency_mean_ms=40)
    tick, jmp, out = run_twins(3, single_key_txn, 0.7, oracle=oracle_of(3, **kw), **kw)
    assert out[:3] == [O.T["init_ok"]] * 3 and all(r is not None for r in out[3:])


def txn_tree_timeouts(s, body):
    from test_txn_tree import txn_ops
    n = 3
    s.add_endpoint("lin-kv", O.KIND_SERVICE)
    s.add_endpoint("lww-kv", O.KIND_SERVICE)
    cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(3)]
    s.schedule(ops_array([(0, cs[i], i, "init", 1, 0) for i in range(n)]))
    rng = np.random.default_rng(5)
    s.schedule(txn_ops(rng, n, cs, 20, 12, 3, 30, [100] * 3))
    s.run(7_500_000_000)
    return s.client_replies()


def test_txn_tree_promise_timeouts_under_loss():
    kw = dict(workload="txn-list-append-tree", latency_dist="constant", latency_mean_ms=1, p_loss=0.1,
              max_endpoints=19, ring_cap=512, max_window=256, server_ring_cap=128, server_max_window=64, rpc_table=128,
              tree_ptrs=2048, journal_cap_log2=20, calendar_slots=16, calendar_cap=2048, seed=99)
    tick, jmp, _ = run_twins(3, txn_tree_timeouts, 0.5, oracle=oracle_of(3, **kw), **kw)
    sends = (jmp["ev"]["event_id"] >> np.uint64(63)) == 0
    errs = jmp["bd"][(jmp["bd"]["type"] == O.T["error"]) & sends & (jmp["ev"]["src"] < 3)]
    assert 0 in set(int(c) for c in errs["p0"])       # a promise timed out after 5 s of idle ticks


# ----------------------------------------------------------------------------------------------- host endpoints
def test_client_rpc_timeout_and_recv_json():
    import maelstrom_b200 as mb
    from maelstrom_b200 import client as Cl
    from maelstrom_b200.engine import KIND_HOST
    from maelstrom_b200.net import Net
    res = []
    for jump in (False, True):
        s = mb.Sim(3, workload="echo", max_endpoints=16)
        if jump:
            s.idle_jump()
        net = Net(s, mb.body)
        c = Cl.Client(net)
        got = [c.rpc("n0", {"type": "init", "node_id": "n0", "node_ids": ["n0", "n1", "n2"]})["type"]]
        try:
            c.rpc("n1", {"type": "no-such-rpc"})             # echo.rb answers nothing it does not know: 5 s timeout
            got.append("answered")
        except Exception as e:                             # noqa: BLE001 -- the client's timeout, whatever its class
            got.append(type(e).__name__)
        got.append((s.now, s.round))
        # ms_recv_json on a host endpoint: a request, its reply as the line a node reads, then a wait with nothing
        h = s.add_endpoint("h0", KIND_HOST)
        s.L.ms_send_json(s.h, json.dumps({"src": "h0", "dest": "n2", "body": {"type": "echo", "msg_id": 7}}).encode())
        buf = C.create_string_buffer(4096)
        assert s.L.ms_recv_json(s.h, h, 50 * MS, buf, 4096) == 1
        got.append(json.loads(buf.value.decode())["body"]["type"])
        assert s.L.ms_recv_json(s.h, h, 2500 * MS + 300_000, buf, 4096) == 0
        got.append((s.now, s.round, s.counters()["rounds"] < s.round if jump else True))
        ev, bd = s.drain()
        res.append((got, ev.tobytes(), bd.tobytes(), s.stats()))
        s.close()
    assert res[0] == res[1]
    assert res[1][0][1] != "answered" and res[1][0][2][0] >= 5000 * MS


# ----------------------------------------------------------------------------------------------- journal paths
@pytest.mark.parametrize("fmt", [32, 8, 4])
def test_streamed_journal_jumps_across_batches(fmt):
    import maelstrom_b200 as mb
    res = []
    for jump in (False, True):
        s = mb.Sim(5, workload="broadcast", topology="line", latency_dist="constant", latency_mean_ms=30,
                   max_endpoints=8, ring_cap=64, max_window=64, calendar_slots=64, calendar_cap=1024, history_rounds=128)
        if jump:
            s.idle_jump()
        c = s.add_endpoint("c0", O.KIND_SIM_CLIENT)
        s.schedule(ops_array([(t * MS, c, t % 5, "broadcast", i + 1, i) for i, t in enumerate(range(0, 3000, 170))]))
        batches = []
        for until in (900 * MS, 1700 * MS + 123, 3200 * MS):
            s.run_streamed(until, sink=lambda info, rows, ev: batches.append(ev.tobytes()), fmt=fmt, decode=True)
        res.append((b"".join(batches), s.now, s.round, s.stats(), s.client_replies(), s.counters()["rounds"]))
        s.close()
    assert res[0][:5] == res[1][:5] and len(res[0][0]) > 0
    assert res[1][5] * 4 < res[0][5]


def small_history(s, body):
    c = s.add_endpoint("c0", O.KIND_SIM_CLIENT)
    # (an idle stretch longer than the history stalls ticking too: the drain only moves on over rounds with events)
    s.schedule(ops_array([(t * MS, c, t % 4, "broadcast", i + 1, i) for i, t in enumerate(range(0, 2000, 45))]))
    s.run(2010 * MS)                                  # Sim.run drains whenever the device asks for it
    return s.now


def test_small_history_meets_back_pressure():
    kw = dict(workload="broadcast", topology="total", latency_dist="constant", latency_mean_ms=5, max_endpoints=8,
              ring_cap=64, max_window=64, calendar_slots=16, calendar_cap=512, history_rounds=64)
    run_twins(4, small_history, 0.6, oracle=oracle_of(4, **kw), **kw)


# ----------------------------------------------------------------------------------------------- wheel edges
def lapping(s, body):
    c = s.add_endpoint("c0", O.KIND_SIM_CLIENT)
    s.schedule(ops_array([(0, c, 0, "broadcast", 1, 1), (10 * MS, c, 3, "broadcast", 2, 2)]))
    s.run(250 * MS + 17)                              # not on a tick boundary
    s.slow()                                          # 10 x: 900 ms in flight, several laps of 64 slots
    s.schedule(ops_array([(300 * MS, c, 1, "broadcast", 3, 3)]))
    s.run(2900 * MS + 1)
    s.fast()
    s.schedule(ops_array([(3000 * MS, c, 2, "broadcast", 4, 4)]))
    s.run(3700 * MS + 999_999)
    return [s.node_set(k).tolist() for k in range(4)]


def test_wheel_laps_slow_fast_and_odd_until():
    kw = dict(workload="broadcast", topology="line", latency_dist="constant", latency_mean_ms=90, max_endpoints=8,
              ring_cap=64, max_window=64, calendar_slots=64, calendar_cap=1024)
    tick, jmp, sets = run_twins(4, lapping, 0.8, oracle=oracle_of(4, **kw), **kw)
    assert all(v == [1, 2, 3, 4] for v in sets)
    assert jmp["now"] == 3701 * MS


# ----------------------------------------------------------------------------------------------- counter origins
def test_origin_below_2_32_rounds():
    kw = dict(workload="echo", max_endpoints=8, ring_cap=64, max_window=64)
    origin = (1 << 32) - 700
    tick, jmp, _ = run_twins(3, sparse_echo, 0.95, origin=origin, **kw)
    assert jmp["round"] > 1 << 32


def test_round_tag_aliasing_across_2_15_rounds():
    # the per-ticket tables are tagged with (round & 0x7FFF) + 1: a jump of more than 2^15 rounds leaves rows that a
    # later round of the same tag reuses; the skipped rows are invalidated, the counts stay exact
    def scenario(s, body):
        c = s.add_endpoint("c0", O.KIND_SIM_CLIENT)
        s.schedule(ops_array([(0, c, 0, "broadcast", 1, 1), (3 * MS, c, 1, "broadcast", 2, 2),
                              (33_000 * MS, c, 2, "broadcast", 3, 3), (33_001 * MS, c, 3, "broadcast", 4, 4),
                              (33_100 * MS, c, 1, "read", 5, 0)]))
        s.run(33_200 * MS)
        return [s.node_set(k).tolist() for k in range(4)]
    kw = dict(workload="broadcast", topology="total", latency_dist="constant", latency_mean_ms=2, max_endpoints=8,
              ring_cap=64, max_window=64, calendar_slots=16, calendar_cap=256, history_rounds=16, journal_level=0)
    tick, jmp, sets = run_twins(4, scenario, 0.99, origin=(1 << 15) - 5, jump_first=True, **kw)
    assert all(v == [1, 2, 3, 4] for v in sets)


# ----------------------------------------------------------------------------------------------- API
def test_step_never_jumps_and_graph_replay_is_refused():
    s = engine(3, workload="echo", max_endpoints=8)
    s.idle_jump()
    r0 = s.round
    s.step(40)
    assert s.round == r0 + 40 and s.counters()["rounds"] == 40
    s.run(3000 * MS)
    assert s.now == 3000 * MS and s.counters()["rounds"] < 60
    s.idle_jump(False)
    s.run(3100 * MS)
    assert s.counters()["rounds"] >= 140
    s.close()
    g = engine(3, workload="echo", max_endpoints=8, use_graph=1)
    assert g.L.ms_set_idle_jump(g.h, 1) == -2
    assert g.L.ms_set_idle_jump(g.h, 0) == 0
    g.close()


def test_sharded_simulation_refuses_the_jump(engine_backend):
    if engine_backend != "emul":
        pytest.skip("sharding in one process is the emulator's (tests/test_emul_sharded.py)")
    import maelstrom_b200 as mb
    shards = [mb.Sim(8, workload="echo", max_endpoints=16, n_shards=2, shard_id=k) for k in range(2)]
    for s in shards:
        assert s.L.ms_set_idle_jump(s.h, 1) == -2
        assert "shard" in s.L.ms_last_error(s.h).decode()
        s.close()


# ----------------------------------------------------------------------------------------------- concurrent CTAs
@pytest.mark.parametrize("seed", [3])
def test_concurrent_ctas(engine_backend, monkeypatch, seed):
    if engine_backend != "emul":
        pytest.skip("the emulator's CTA interleaving; the GPU has concurrent CTAs in every case above")
    import emul_lib
    L = emul_lib.load()
    L.simt_ctas.argtypes = [C.c_longlong]
    monkeypatch.setenv("MS_EMUL_SMS", "4")
    L.simt_ctas(seed)
    try:
        kw = dict(workload="broadcast", topology="grid", n_values=1 << 10, latency_dist="exponential",
                  latency_mean_ms=100, p_loss=0.05, max_endpoints=600, ring_cap=256, max_window=128,
                  calendar_slots=256, calendar_cap=4096, seed=11)
        run_twins(9, broadcast_clients, 0.2, oracle=oracle_of(9, **kw), **kw)
        kw = dict(workload="g-set", latency_dist="constant", latency_mean_ms=20, n_values=64, max_endpoints=600,
                  ring_cap=64, max_window=64, calendar_slots=64, calendar_cap=1024)
        run_twins(4, gset_periodic, 0.95, oracle=oracle_of(4, **kw), **kw)
    finally:
        L.simt_ctas(int(os.environ.get("MS_EMUL_CTAS", "-1") or -1))
