"""Scenarios run identically against the oracle (tests/oracle_lib.Sim) and the
CUDA engine (maelstrom_b200.Sim): both expose the same method names."""
import numpy as np

import oracle_lib as O


def make_pair(n_nodes, **kw):
    """Create (engine, oracle) with identical configuration."""
    import maelstrom_b200 as mb
    sizing = {k: kw.pop(k) for k in list(kw) if k in (
        "max_endpoints", "ring_cap", "max_window", "journal_cap_log2", "journal_level",
        "calendar_slots", "calendar_cap", "mailbox_cap", "inject_cap", "threads_per_node",
        "n_keys", "raft_log_cap", "history_rounds", "server_ring_cap", "server_max_window")}
    workload = kw.pop("workload", "broadcast")
    g = mb.Sim(n_nodes, workload=workload, **kw, **sizing)
    o = O.Sim(n_nodes, workload={"echo": O.W_ECHO, "broadcast": O.W_BROADCAST, "g-set": O.W_GSET, "lin-kv": O.W_RAFT, "txn-list-append": O.W_TXN,
                                 "txn-list-append-tree": O.W_TXN_TREE}[workload], **kw)
    return g, o


def both(g, o, fn):
    """Apply fn(sim, body_factory) to both and assert equal results."""
    import maelstrom_b200 as mb
    rg = fn(g, mb.body)
    ro = fn(o, O.body)
    return rg, ro


def assert_same_journal(g, o):
    ev_g, bd_g = g.drain()
    ev_o, bd_o = o.journal()
    assert len(ev_g) == len(ev_o), (len(ev_g), len(ev_o))
    for f in ("event_id", "time_ns", "msg_id", "src", "dest"):
        if not np.array_equal(ev_g[f], ev_o[f]):
            bad = int(np.nonzero(ev_g[f] != ev_o[f])[0][0])
            raise AssertionError("journal field %s differs first at event %d: gpu=%s oracle=%s" %
                                 (f, bad, ev_g[bad], ev_o[bad]))
    for f in ("type", "flags", "msg_id", "in_reply_to", "p0", "p1"):
        if not np.array_equal(bd_g[f], bd_o[f]):
            bad = int(np.nonzero(bd_g[f] != bd_o[f])[0][0])
            raise AssertionError("body field %s differs first at event %d: gpu=%s oracle=%s" %
                                 (f, bad, bd_g[bad], bd_o[bad]))
    assert np.array_equal(bd_g["id"], ev_g["msg_id"])
    assert g.stats() == o.stats()
    assert g.now == o.now and g.round == o.round
    return ev_g, bd_g


def oracle_gossip_sends(ev, bd, n_nodes):
    """Server -> server broadcast gossip in an oracle journal (level 2: events and bodies): the :send events
    with src and dest < n_nodes, type broadcast and no reply flag.  These are the messages the engine may
    carry as 16-B compact records."""
    send = (ev["event_id"] & np.uint64(O.RECV_BIT)) == 0
    gossip = (send & (ev["src"] < n_nodes) & (ev["dest"] < n_nodes) & (bd["type"] == O.T["broadcast"]) &
              ((bd["flags"] & O.F_REPLY) == 0))
    return int(np.count_nonzero(gossip))


def compact_total(rc):
    """Records claimed on all compact rings so far (Sim.ring_counters(); counters start at 0 and wrap)."""
    return int(rc["ctail"].astype(np.uint64).sum())


def compact_delta(rc1, rc0):
    """Compact records claimed between two ring_counters() reads, per server (modulo 2^32)."""
    return (rc1["ctail"] - rc0["ctail"]).astype(np.uint32)


def ops_array(rows):
    """rows: (time_ns, src, dest, type, msg_id, p0)"""
    a = np.zeros(len(rows), dtype=O.OP_DTYPE)
    for i, (t, s, d, ty, mid, p0) in enumerate(rows):
        a[i]["time_ns"] = t
        a[i]["src"] = s
        a[i]["dest"] = d
        a[i]["body"]["type"] = O.T[ty]
        a[i]["body"]["flags"] = O.F_MSG_ID
        a[i]["body"]["msg_id"] = mid
        a[i]["body"]["p0"] = p0
    return a


def random_broadcast_ops(n_nodes, clients, n_ticks, per_tick, seed=7, tick_ns=1_000_000):
    rng = np.random.default_rng(seed)
    rows = []
    mid = {c: 0 for c in clients}
    v = 0
    for t in range(n_ticks):
        for _ in range(per_tick):
            c = clients[int(rng.integers(len(clients)))]
            mid[c] += 1
            rows.append((t * tick_ns, c, int(rng.integers(n_nodes)), "broadcast", mid[c], v))
            v += 1
    return ops_array(rows), v
