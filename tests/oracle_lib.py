"""ctypes binding of the CPU oracle (oracle/_build/liboracle.so).

Test infrastructure only: imported by tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline / --impl reference legs.  Never imported by the
product package (maelstrom_b200/).
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ORACLE_DIR = os.path.join(os.path.dirname(_HERE), "oracle")
_SO = os.path.join(_ORACLE_DIR, "_build", "liboracle.so")

MSG_DTYPE = np.dtype([("id", "<u8"), ("deadline_ns", "<i8"), ("src", "<u4"), ("dest", "<u4"),
                      ("msg_id", "<u4"), ("in_reply_to", "<u4"), ("type", "<u2"), ("flags", "<u2"),
                      ("p0", "<u4"), ("p1", "<u8")])
EVENT_DTYPE = np.dtype([("event_id", "<u8"), ("time_ns", "<i8"), ("msg_id", "<u8"),
                        ("src", "<u4"), ("dest", "<u4")])
BODY_DTYPE = np.dtype([("type", "<u2"), ("flags", "<u2"), ("msg_id", "<u4"), ("in_reply_to", "<u4"),
                       ("p0", "<u4"), ("p1", "<u8")])
OP_DTYPE = np.dtype([("time_ns", "<i8"), ("src", "<u4"), ("dest", "<u4"), ("body", BODY_DTYPE)])
assert MSG_DTYPE.itemsize == 48 and EVENT_DTYPE.itemsize == 32
assert BODY_DTYPE.itemsize == 24 and OP_DTYPE.itemsize == 40

W_ECHO, W_BROADCAST, W_GSET, W_RAFT, W_TXN, W_TXN_TREE = 0, 1, 2, 3, 4, 5
TOPO = {"grid": 0, "line": 1, "total": 2, "tree": 3, "tree2": 3, "tree3": 4, "tree4": 5}
DIST = {"constant": 0, "uniform": 1, "exponential": 2}
KIND_SERVER, KIND_CLIENT, KIND_HOST, KIND_SIM_CLIENT, KIND_SERVICE, KIND_GEN_CLIENT = 0, 1, 2, 3, 4, 5
HIST_DTYPE = np.dtype([("time_ns", "<i8"), ("order", "<u8"), ("client", "<u4"), ("op", "<u4"), ("type", "u1"),
                       ("f", "u1"), ("error", "<u2"), ("value", "<u4")])


class GenConfig(C.Structure):
    _fields_ = [("n_clients", C.c_uint32), ("read_permille", C.c_uint32), ("interval_ns", C.c_int64),
                ("timeout_ns", C.c_int64), ("time_limit_ns", C.c_int64), ("quiet_ns", C.c_int64)]
SVC = {"lin-kv": 0, "seq-kv": 1, "lww-kv": 2, "lin-tso": 3}
T = dict(init=1, init_ok=2, error=3, echo=10, echo_ok=11, topology=20, topology_ok=21,
         broadcast=22, broadcast_ok=23, read=24, read_ok=25, add=30, add_ok=31,
         replicate_one=32, replicate_full=33, write=40, write_ok=41, cas=42, cas_ok=43, ts=44, ts_ok=45,
         request_vote=50, request_vote_res=51, append_entries=52, append_entries_res=53,
         txn=60, txn_ok=61)
F_MSG_ID, F_REPLY, F_CREATE, F_APPENDS = 1, 2, 4, 8
RECV_BIT = 1 << 63


class Config(C.Structure):
    _fields_ = [("n_nodes", C.c_uint32), ("workload", C.c_uint32), ("topology", C.c_uint32),
                ("latency_dist", C.c_uint32), ("latency_mean_ms", C.c_uint32),
                ("seed_lo", C.c_uint32), ("seed_hi", C.c_uint32), ("p_loss", C.c_double),
                ("n_values", C.c_uint32), ("gset_interval_ms", C.c_uint32),
                ("raft_group", C.c_uint32), ("rpc_table", C.c_uint32), ("tree_ptrs", C.c_uint32)]


class Body(C.Structure):
    _fields_ = [("type", C.c_uint16), ("flags", C.c_uint16), ("msg_id", C.c_uint32),
                ("in_reply_to", C.c_uint32), ("p0", C.c_uint32), ("p1", C.c_uint64)]


def build():
    subprocess.check_call(["make", "-s", "-C", _ORACLE_DIR])


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(
                os.path.join(_ORACLE_DIR, "oracle.cpp")):
            build()
        L = C.CDLL(_SO)
        L.or_create.restype = C.c_void_p
        L.or_tree_key_hash.restype = C.c_uint32
        L.or_tree_key_hash.argtypes = [C.c_uint32]
        L.or_create.argtypes = [C.POINTER(Config)]
        L.or_destroy.argtypes = [C.c_void_p]
        L.or_last_error.restype = C.c_char_p
        L.or_last_error.argtypes = [C.c_void_p]
        L.or_add_endpoint.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
        L.or_remove_endpoint.argtypes = [C.c_void_p, C.c_uint32]
        L.or_send.restype = C.c_int64
        L.or_send.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(Body)]
        L.or_schedule.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
        L.or_step.argtypes = [C.c_void_p, C.c_uint64]
        L.or_run.argtypes = [C.c_void_p, C.c_int64]
        L.or_recv.argtypes = [C.c_void_p, C.c_uint32, C.c_int64, C.c_void_p]
        L.or_now.restype = C.c_int64
        L.or_now.argtypes = [C.c_void_p]
        L.or_round.restype = C.c_uint64
        L.or_round.argtypes = [C.c_void_p]
        L.or_set_origin.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64]
        L.or_net_drop.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
        for f in ("or_net_heal", "or_net_slow", "or_net_fast", "or_net_flaky"):
            getattr(L, f).argtypes = [C.c_void_p]
        L.or_net_set_loss.argtypes = [C.c_void_p, C.c_double]
        L.or_net_partition.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
        L.or_journal_size.restype = C.c_size_t
        L.or_journal_size.argtypes = [C.c_void_p]
        L.or_journal_copy.restype = C.c_size_t
        L.or_journal_copy.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t]
        L.or_stats.argtypes = [C.c_void_p, C.c_void_p]
        L.or_node_set.restype = C.c_size_t
        L.or_node_set.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t]
        L.or_read_snapshot.restype = C.c_size_t
        L.or_read_snapshot.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_size_t]
        L.or_client_replies.restype = C.c_uint64
        L.or_client_replies.argtypes = [C.c_void_p]
        L.or_add_gen_clients.argtypes = [C.c_void_p, C.POINTER(GenConfig), C.c_uint32]
        L.or_history_copy.restype = C.c_size_t
        L.or_history_copy.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
        L.or_undeliverable.restype = C.c_uint64
        L.or_undeliverable.argtypes = [C.c_void_p]
        L.or_topology.restype = C.c_size_t
        L.or_topology.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t]
        L.or_philox4x32_10.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.or_latency_draw.restype = C.c_uint64
        L.or_latency_draw.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]
        L.or_loss_threshold.restype = C.c_uint64
        L.or_loss_threshold.argtypes = [C.c_double]
        L.or_raft_state.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
        L.or_raft_append.argtypes = [C.c_void_p, C.c_uint32, C.c_uint64, C.c_void_p]
        L.or_service_new.restype = C.c_void_p
        L.or_service_new.argtypes = [C.c_int, C.c_uint32]
        L.or_service_free.argtypes = [C.c_void_p]
        L.or_service_handle.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(Body), C.c_uint32, C.POINTER(Body)]
        _lib = L
    return _lib


def topology(name, n, node):
    out = np.zeros(max(n, 4), dtype=np.uint32)
    k = lib().or_topology(TOPO[name], n, node, out.ctypes.data, out.size)
    return out[:k].tolist()


def philox(ctr, key):
    c = np.asarray(ctr, dtype=np.uint32)
    k = np.asarray(key, dtype=np.uint32)
    o = np.zeros(4, dtype=np.uint32)
    lib().or_philox4x32_10(c.ctypes.data, k.ctypes.data, o.ctypes.data)
    return o.tolist()


def latency_draw(dist, mean_ms, scale, x):
    xs = np.asarray(x, dtype=np.uint32)
    return int(lib().or_latency_draw(DIST[dist], mean_ms, scale, xs.ctypes.data))


def body(type, msg_id=None, in_reply_to=None, p0=0, p1=0, create=False, appends=False):
    b = Body()
    b.type = T[type] if isinstance(type, str) else type
    b.flags = ((F_MSG_ID if msg_id is not None else 0) | (F_REPLY if in_reply_to is not None else 0) |
               (F_CREATE if create else 0) | (F_APPENDS if appends else 0))
    b.msg_id = msg_id or 0
    b.in_reply_to = in_reply_to or 0
    b.p0 = p0
    b.p1 = p1
    return b


class Sim:
    """Thin object wrapper; method names follow the C ABI (include/maelstrom_b200.h)."""

    def __init__(self, n_nodes, workload=W_BROADCAST, topology="grid", latency_dist="constant",
                 latency_mean_ms=0, seed=0x4D41454C, p_loss=0.0, n_values=1 << 16, gset_interval_ms=5000,
                 raft_group=0, rpc_table=0, tree_ptrs=0):
        cfg = Config()
        cfg.n_nodes = n_nodes
        cfg.workload = workload
        cfg.topology = TOPO[topology]
        cfg.latency_dist = DIST[latency_dist]
        cfg.latency_mean_ms = latency_mean_ms
        cfg.seed_lo = seed & 0xFFFFFFFF
        cfg.seed_hi = seed >> 32
        cfg.p_loss = p_loss
        cfg.n_values = n_values
        cfg.gset_interval_ms = gset_interval_ms
        cfg.raft_group = raft_group
        cfg.rpc_table = rpc_table
        cfg.tree_ptrs = tree_ptrs
        self.L = lib()
        self.h = self.L.or_create(C.byref(cfg))
        self.n_nodes = n_nodes
        self.workload = int(workload)

    def close(self):
        if self.h:
            self.L.or_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def _chk(self, rc):
        if rc < 0:
            raise RuntimeError("oracle error %d: %s" % (rc, self.L.or_last_error(self.h).decode()))
        return rc

    def add_endpoint(self, name, kind=KIND_CLIENT):
        return self._chk(self.L.or_add_endpoint(self.h, name.encode(), kind))

    def remove_endpoint(self, idx):
        return self.L.or_remove_endpoint(self.h, idx)

    def send(self, src, dest, b):
        return self.L.or_send(self.h, src, dest, C.byref(b))

    def schedule(self, ops):
        ops = np.ascontiguousarray(ops, dtype=OP_DTYPE)
        return self._chk(self.L.or_schedule(self.h, ops.ctypes.data, ops.size))

    def step(self, n=1):
        return self._chk(self.L.or_step(self.h, n))

    def run(self, until_ns):
        return self._chk(self.L.or_run(self.h, until_ns))

    def recv(self, endpoint, timeout_ns=0):
        out = np.zeros(1, dtype=MSG_DTYPE)
        rc = self._chk(self.L.or_recv(self.h, endpoint, timeout_ns, out.ctypes.data))
        return out[0] if rc == 1 else None

    @property
    def now(self):
        return self.L.or_now(self.h)

    @property
    def round(self):
        return self.L.or_round(self.h)

    def set_origin(self, round=0, msg_id=0, event_id=0, ring_pos=0, ring_stride=0):
        """or_set_origin; ring_pos / ring_stride are the engine's and have no oracle counterpart."""
        return self._chk(self.L.or_set_origin(self.h, round, msg_id, event_id))

    def drop(self, src, dest):
        return self.L.or_net_drop(self.h, src, dest)

    def heal(self):
        return self.L.or_net_heal(self.h)

    def slow(self):
        return self.L.or_net_slow(self.h)

    def fast(self):
        return self.L.or_net_fast(self.h)

    def flaky(self):
        return self.L.or_net_flaky(self.h)

    def set_loss(self, p):
        return self.L.or_net_set_loss(self.h, p)

    def partition(self, comp):
        comp = np.ascontiguousarray(comp, dtype=np.uint32)
        return self.L.or_net_partition(self.h, comp.ctypes.data, comp.size)

    def journal(self):
        n = self.L.or_journal_size(self.h)
        ev = np.zeros(n, dtype=EVENT_DTYPE)
        bd = np.zeros(n, dtype=BODY_DTYPE)
        got = self.L.or_journal_copy(self.h, 0, ev.ctypes.data, bd.ctypes.data, n)
        assert got == n
        return ev, bd

    def stats(self):
        out = np.zeros(9, dtype=np.uint64)
        self.L.or_stats(self.h, out.ctypes.data)
        keys = ("send-count", "recv-count", "msg-count")
        return {cls: {k: int(out[i * 3 + j]) for j, k in enumerate(keys)}
                for i, cls in enumerate(("all", "clients", "servers"))}

    def node_set(self, node):
        n = self.L.or_node_set(self.h, node, None, 0)
        out = np.zeros(n, dtype=np.uint32)
        self.L.or_node_set(self.h, node, out.ctypes.data, n)
        return out

    def read_snapshot(self, msg_id):
        n = self.L.or_read_snapshot(self.h, msg_id, None, 0)
        out = np.zeros(n, dtype=np.uint32)
        self.L.or_read_snapshot(self.h, msg_id, out.ctypes.data, n)
        return out

    RAFT_FIELDS = ("state", "term", "voted_for", "commit_index", "last_applied", "leader", "log_size", "kv_size")

    def raft_state(self, node):
        """state 0 nascent / 1 follower / 2 candidate / 3 leader; voted_for and leader are -1 when unset"""
        out = np.zeros(8, dtype=np.uint64)
        self._chk(self.L.or_raft_state(self.h, node, out.ctypes.data))
        d = dict(zip(self.RAFT_FIELDS, (int(x) for x in out)))
        d["voted_for"] -= 1
        d["leader"] -= 1
        return d

    def client_replies(self):
        return int(self.L.or_client_replies(self.h))

    def undeliverable(self):
        return int(self.L.or_undeliverable(self.h))

    def add_gen_clients(self, n_clients, interval_ns, time_limit_ns, read_permille=500, timeout_ns=0, quiet_ns=0,
                        first_name=0):
        gc = GenConfig(n_clients, read_permille, interval_ns, timeout_ns, time_limit_ns, quiet_ns)
        return self._chk(self.L.or_add_gen_clients(self.h, C.byref(gc), first_name))

    def history(self):
        """everything since the last call (the engine's ms_history_drain has the same contract)"""
        first = getattr(self, "_hist_seen", 0)
        n = self.L.or_history_copy(self.h, first, None, 0)
        out = np.zeros(n, dtype=HIST_DTYPE)
        if n:
            self.L.or_history_copy(self.h, first, out.ctypes.data, n)
        self._hist_seen = first + n
        return out


class Service:
    """One service on its own (oracle's restatement of service.clj), driven the way
    test/maelstrom/service_test.clj drives handle!; rnd = the 32-bit draw behind rand-int."""

    def __init__(self, name, buffer_size=0):
        self.L = lib()
        self.h = self.L.or_service_new(SVC[name], buffer_size)

    def __del__(self):
        if getattr(self, "h", None):
            self.L.or_service_free(self.h)
            self.h = None

    def handle(self, client, req, rnd=0):
        out = Body()
        if not self.L.or_service_handle(self.h, client, C.byref(req), rnd & 0xFFFFFFFF, C.byref(out)):
            return None
        return out
