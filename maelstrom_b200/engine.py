"""Object wrapper over the C ABI (include/maelstrom_b200.h).  Method names
follow the ABI entry points, which in turn follow maelstrom.net's public
functions (src/maelstrom/net.clj:79-247)."""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import Body, Config, EVENT_DTYPE, JBODY_DTYPE, MSG_DTYPE, OP_DTYPE  # noqa: F401

WORKLOADS = {"echo": 0, "broadcast": 1, "g-set": 2, "lin-kv": 3, "txn-list-append": 4, "txn-list-append-tree": 5,
             "lin-kv-proxy": 6, "kafka": 7, "g-counter": 8, "pn-counter": 9, "txn-rw-register": 10}
TOPOLOGIES = {"grid": 0, "line": 1, "total": 2, "tree": 3, "tree2": 3, "tree3": 4, "tree4": 5}
DISTS = {"constant": 0, "uniform": 1, "exponential": 2}
KIND_SERVER, KIND_CLIENT, KIND_HOST, KIND_SIM_CLIENT, KIND_SERVICE = 0, 1, 2, 3, 4
SERVICES = ("lin-kv", "seq-kv", "lww-kv", "lin-tso")      # service/default-services, service.clj:290-296
TYPES = dict(init=1, init_ok=2, error=3, echo=10, echo_ok=11, topology=20, topology_ok=21,
             broadcast=22, broadcast_ok=23, read=24, read_ok=25, add=30, add_ok=31,
             replicate_one=32, replicate_full=33, write=40, write_ok=41, cas=42, cas_ok=43, ts=44, ts_ok=45,
             request_vote=50, request_vote_res=51, append_entries=52, append_entries_res=53,
             txn=60, txn_ok=61)
# the kafka workload's types (MS_T_SEND ...): the device's own encoding, unknown to the JSON envelope and the oracle
KAFKA_TYPES = dict(send=70, send_ok=71, poll=72, poll_ok=73, commit_offsets=74, commit_offsets_ok=75,
                   list_committed_offsets=76, list_committed_offsets_ok=77)
# the counter workloads' merge / merge_ok (MS_T_MERGE ...): the device's own encoding, as kafka's
COUNTER_TYPES = dict(merge=80, merge_ok=81)
# the txn-rw-register node's replicate / replicate_ack (MS_T_REPLICATE ...): the device's own encoding, as kafka's
TXN_RW_TYPES = dict(replicate=90, replicate_ack=91)
TYPE_NAMES = {v: k for k, v in TYPES.items()}
F_MSG_ID, F_REPLY, F_CREATE, F_APPENDS = 1, 2, 4, 8
RECV_BIT = 1 << 63


class SimError(RuntimeError):
    def __init__(self, code, text):
        RuntimeError.__init__(self, "maelstrom_b200 error %d: %s" % (code, text))
        self.code = code


def body(type, msg_id=None, in_reply_to=None, p0=0, p1=0, create=False, appends=False):
    b = Body()
    b.type = {**TYPES, **KAFKA_TYPES, **COUNTER_TYPES, **TXN_RW_TYPES}[type] if isinstance(type, str) else type
    b.flags = ((F_MSG_ID if msg_id is not None else 0) | (F_REPLY if in_reply_to is not None else 0) |
               (F_CREATE if create else 0) | (F_APPENDS if appends else 0))
    b.msg_id = msg_id or 0
    b.in_reply_to = in_reply_to or 0
    b.p0 = p0
    b.p1 = p1
    return b


class JournalDecoder:
    """ms_jdecoder: expands MS_JFMT_4 batches (32 bits per event) into EVENT_DTYPE records.  It follows the
    stream: a :recv's src / dest are those of the :send with the same id, seen earlier."""

    def __init__(self, log2_window=22):
        self.L = _lib.lib()
        self.h = self.L.ms_jdecoder_create(log2_window)
        if not self.h:
            raise MemoryError("ms_jdecoder_create")

    def close(self):
        if self.h:
            self.L.ms_jdecoder_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def _chk(self, rc):
        if rc < 0:
            raise SimError(rc, self.L.ms_jdecoder_error(self.h).decode())

    def decode_raw(self, batch_p, rounds_p, events_p, n):
        ev = np.zeros(n, dtype=EVENT_DTYPE)
        self._chk(self.L.ms_jdecoder_decode(self.h, batch_p, rounds_p, events_p, ev.ctypes.data))
        return ev

    def note(self, events):
        """events (EVENT_DTYPE) obtained outside the stream, e.g. from Sim.drain()"""
        ev = np.ascontiguousarray(events, dtype=EVENT_DTYPE)
        self._chk(self.L.ms_jdecoder_note(self.h, ev.ctypes.data, len(ev)))


class Sim:
    def __init__(self, n_nodes, workload="broadcast", topology="grid", latency_dist="constant",
                 latency_mean_ms=0, seed=0x4D41454C, p_loss=0.0, n_values=1 << 16, **sizing):
        cfg = Config()
        cfg.n_nodes = n_nodes
        cfg.workload = WORKLOADS[workload] if isinstance(workload, str) else workload
        cfg.topology = TOPOLOGIES[topology]
        cfg.latency_dist = DISTS[latency_dist]
        cfg.latency_mean_ms = latency_mean_ms
        cfg.seed_lo = seed & 0xFFFFFFFF
        cfg.seed_hi = seed >> 32
        cfg.p_loss = p_loss
        cfg.n_values = n_values
        cfg.journal_level = 2
        # lin-kv-proxy: the service the proxies forward to (ms_config.reserved[3], MS_SVC_*)
        if "proxy_service" in sizing:
            name = sizing.pop("proxy_service")
            cfg.reserved[3] = SERVICES.index(name) if isinstance(name, str) else int(name)
        # named spellings of ms_config.reserved[]
        for name, slot in (("history_rounds", 0), ("use_graph", 1), ("n_keys", 2), ("raft_log_cap", 3),
                           ("raft_group", 4), ("rpc_table", 5), ("tree_ptrs", 3), ("tree_cache", 4),
                           ("kafka_keys", 2), ("kafka_log_cap", 3), ("txn_rw_keys", 2), ("txn_rw_log_cap", 3)):
            if name in sizing:
                cfg.reserved[slot] = int(sizing.pop(name))
        for k, v in sizing.items():
            if not hasattr(cfg, k):
                raise TypeError("unknown ms_config field %r" % k)
            setattr(cfg, k, v)
        self.L = _lib.lib()
        self._stash = []
        self.cfg = cfg
        self.n_nodes = n_nodes
        self.workload = int(cfg.workload)
        self.h = self.L.ms_create(C.byref(cfg))
        if not self.h:
            raise SimError(-4, self.L.ms_last_error(None).decode())

    def close(self):
        if getattr(self, "h", None):
            self.L.ms_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _chk(self, rc):
        if rc < 0:
            raise SimError(rc, self.L.ms_last_error(self.h).decode())
        return rc

    # endpoints -----------------------------------------------------------
    def add_endpoint(self, name, kind=KIND_CLIENT):
        return self._chk(self.L.ms_add_endpoint(self.h, name.encode(), kind))

    def remove_endpoint(self, idx):
        return self.L.ms_remove_endpoint(self.h, idx)

    def endpoint_index(self, name):
        return self.L.ms_endpoint_index(self.h, name.encode())

    # data plane ----------------------------------------------------------
    def send(self, src, dest, b):
        return self.L.ms_send(self.h, src, dest, C.byref(b))

    def recv(self, endpoint, timeout_ns=0):
        out = np.zeros(1, dtype=MSG_DTYPE)
        deadline = self.now + timeout_ns
        while True:
            rc = self.L.ms_recv(self.h, endpoint, max(0, deadline - self.now), out.ctypes.data)
            if rc == -5 and self.cfg.journal_level and not self.cfg.journal_discard:
                # MS_ERR_CAPACITY: the device wants the journal drained before it runs more rounds
                # (nothing was executed); stash the events and wait on
                self._stash.append(self._drain_now())
                continue
            self._chk(rc)
            return out[0] if rc == 1 else None

    def add_gen_clients(self, n_clients, interval_ns, time_limit_ns, read_permille=None, timeout_ns=0, quiet_ns=0,
                        first_name=0):
        """ms_add_gen_clients: closed-loop clients on the device; returns the first endpoint index.  read_permille
        defaults to gen/mix's 500, and to 667 on g-counter, whose gen/filter redraws the negative adds"""
        if read_permille is None:
            read_permille = 667 if self.cfg.workload == WORKLOADS["g-counter"] else 500
        gc = _lib.GenConfig(n_clients, read_permille, interval_ns, timeout_ns, time_limit_ns, quiet_ns)
        return self._chk(self.L.ms_add_gen_clients(self.h, C.byref(gc), first_name))

    def add_kv_clients(self, n_clients, interval_ns, time_limit_ns, key_period_ns, keys_per_group=1, value_range=0,
                       timeout_ns=0, first_name=0):
        """ms_add_kv_clients: closed-loop lin-kv clients of the Raft nodes or the lin-kv proxies on the device (groups of 2g per key,
        half of them readers); returns the first endpoint index.  history() returns their records,
        kv_history(records, *sim.kv_groups) sorts them into one history per register"""
        kc = _lib.KvGenConfig(n_clients, value_range, keys_per_group, interval_ns, timeout_ns, time_limit_ns,
                              key_period_ns)
        first = self._chk(self.L.ms_add_kv_clients(self.h, C.byref(kc), first_name))
        g = int(self.cfg.reserved[4])
        self.kv_groups = (first, 2 * (g if 0 < g < self.n_nodes else self.n_nodes))   # first client, clients per group
        return first

    def add_kafka_clients(self, n_clients, interval_ns, time_limit_ns, assign_permille=0, crash_permille=0,
                          timeout_ns=0, first_name=0):
        """ms_add_kafka_clients: closed-loop kafka clients of the single-node logs on the device (client k on server
        k mod n_nodes); returns the first endpoint index.  kafka_history() returns their records; sim.kafka_groups =
        (first client, servers per group g = raft_group, 0 = 1)"""
        kc = _lib.KafkaGenConfig(n_clients, assign_permille, crash_permille, 0, interval_ns, timeout_ns, time_limit_ns)
        first = self._chk(self.L.ms_add_kafka_clients(self.h, C.byref(kc), first_name))
        self.kafka_groups = (first, max(1, int(self.cfg.reserved[4])))
        return first

    def kafka_history(self, cap=1 << 20):
        """ms_kafka_history_drain: the kafka clients' records since the last call, in (time, round, client) order"""
        parts = []
        while True:
            out = np.zeros(cap, dtype=_lib.KAFKA_HIST_DTYPE)
            n = C.c_size_t(0)
            self._chk(self.L.ms_kafka_history_drain(self.h, out.ctypes.data, cap, C.byref(n)))
            parts.append(out[:n.value])
            if n.value < cap:
                break
        return np.concatenate(parts)

    def kafka_log(self, node, key):
        """ms_kafka_log: the messages of node's log of `key`, offset order"""
        n = C.c_size_t(0)
        self._chk(self.L.ms_kafka_log(self.h, node, key, None, 0, C.byref(n)))
        out = np.zeros(n.value, dtype=np.uint32)
        self._chk(self.L.ms_kafka_log(self.h, node, key, out.ctypes.data, n.value, C.byref(n)))
        return out

    def kafka_committed(self, node, key):
        """ms_kafka_committed: node's committed offset of `key`, None when nothing is committed"""
        c = self.L.ms_kafka_committed(self.h, node, key)
        return None if c == -1 else self._chk(c)

    def counter_state(self, node):
        """ms_counter_state: node's counter as (inc, dec), int64 arrays with one entry per member of its block"""
        n = self._chk(self.L.ms_counter_state(self.h, node, None, 0))
        out = np.zeros(n, dtype=np.int64)
        self._chk(self.L.ms_counter_state(self.h, node, out.ctypes.data, n))
        return out[:n // 2], out[n // 2:]

    def add_txn_rw_clients(self, n_clients, interval_ns, time_limit_ns, key_period_ns, key_count=1, min_len=1, max_len=4,
                           timeout_ns=0, first_name=0):
        """ms_add_txn_rw_clients: closed-loop txn-rw-register clients on the device (client k on server k mod n_nodes);
        returns the first endpoint index.  txn_rw_history() returns their records"""
        rc = _lib.TxnRwGenConfig(n_clients, min_len, max_len, key_count, interval_ns, timeout_ns, time_limit_ns,
                                 key_period_ns)
        return self._chk(self.L.ms_add_txn_rw_clients(self.h, C.byref(rc), first_name))

    def txn_rw_history(self, cap=1 << 20):
        """ms_txn_rw_history_drain: the txn-rw-register clients' records since the last call, in (time, round, client)
        order"""
        parts = []
        while True:
            out = np.zeros(cap, dtype=_lib.TXN_RW_HIST_DTYPE)
            n = C.c_size_t(0)
            self._chk(self.L.ms_txn_rw_history_drain(self.h, out.ctypes.data, cap, C.byref(n)))
            parts.append(out[:n.value])
            if n.value < cap:
                break
        return np.concatenate(parts)

    def txn_rw_log(self, node):
        """ms_txn_rw_log: node's completed txns in log order (TXN_RW_ENTRY_DTYPE)"""
        n = self._chk(self.L.ms_txn_rw_log(self.h, node, None, 0))
        out = np.zeros(n, dtype=_lib.TXN_RW_ENTRY_DTYPE)
        self._chk(self.L.ms_txn_rw_log(self.h, node, out.ctypes.data, n))
        return out

    def txn_rw_state(self, node):
        """ms_txn_rw_state: (lamport, log length, values, timestamps) of node; values[k] = 0 is nil, ts[k] the lamport
        of the write"""
        lamport, n = C.c_uint64(0), C.c_uint32(0)
        k = self._chk(self.L.ms_txn_rw_state(self.h, node, None, None, None, None, 0))
        val, ts = np.zeros(k, dtype=np.uint32), np.zeros(k, dtype=np.uint64)
        self._chk(self.L.ms_txn_rw_state(self.h, node, C.byref(lamport), C.byref(n), val.ctypes.data, ts.ctypes.data, k))
        return lamport.value, n.value, val, ts

    def history(self, cap=1 << 20):
        """ms_history_drain: the history records since the last call, in (time, round, client) order"""
        parts = []
        while True:
            out = np.zeros(cap, dtype=_lib.HIST_DTYPE)
            n = C.c_size_t(0)
            self._chk(self.L.ms_history_drain(self.h, out.ctypes.data, cap, C.byref(n)))
            parts.append(out[:n.value])
            if n.value < cap:
                break
        return np.concatenate(parts)

    def schedule(self, ops):
        ops = np.ascontiguousarray(ops, dtype=OP_DTYPE)
        return self._chk(self.L.ms_schedule_ops(self.h, ops.ctypes.data, ops.size))

    # time ----------------------------------------------------------------
    def step(self, n=1):
        rc = self.L.ms_step(self.h, n)
        if rc == -5 and self.cfg.journal_level and not self.cfg.journal_discard and n == 1:
            self._stash.append(self._drain_now())     # see recv()
            rc = self.L.ms_step(self.h, n)
        return self._chk(rc)

    def run_raw(self, until_ns):
        """ms_run as is: 0 = reached until_ns, 1 = journal ring half full (drain, then call again)."""
        return self._chk(self.L.ms_run(self.h, until_ns))

    def run(self, until_ns):
        """ms_run; when the device asks for a journal drain, stash the events and continue."""
        while self.run_raw(until_ns) == 1:
            self._stash.append(self._drain_now())
        return 0

    def idle_jump(self, enable=True):
        """ms_set_idle_jump: ms_run / ms_run_streamed / ms_recv jump over ticks at which no endpoint acts, with
        byte-identical outputs; counters() counts only the rounds executed"""
        return self._chk(self.L.ms_set_idle_jump(self.h, 1 if enable else 0))

    @property
    def now(self):
        return self.L.ms_now(self.h)

    @property
    def round(self):
        return self.L.ms_round(self.h)

    # faults --------------------------------------------------------------
    def drop(self, src, dest):
        return self._chk(self.L.ms_net_drop(self.h, src, dest))

    def heal(self):
        return self._chk(self.L.ms_net_heal(self.h))

    def slow(self):
        return self._chk(self.L.ms_net_slow(self.h))

    def fast(self):
        return self._chk(self.L.ms_net_fast(self.h))

    def flaky(self):
        return self._chk(self.L.ms_net_flaky(self.h))

    def set_loss(self, p):
        return self._chk(self.L.ms_net_set_loss(self.h, p))

    def partition(self, comp):
        comp = np.ascontiguousarray(comp, dtype=np.uint32)
        return self._chk(self.L.ms_net_partition(self.h, comp.ctypes.data, comp.size))

    def nemesis(self, time_limit_ns, interval_ns=0, start_ns=None, targets=0, group=0):
        """ms_set_nemesis: a Jepsen partition schedule per cluster, run on the device before every round (DESIGN.md
        2.13).  targets: a mask of NEM_ONE / NEM_MAJORITY / NEM_MINORITY_THIRD / NEM_MAJORITIES_RING (0 = the first
        three); interval_ns 0 = 10 s; start_ns None = now (an earlier instant is refused); group 0 = the workload's
        clusters.  Each op is a history() record with client H_NEMESIS.  With NEM_MAJORITIES_RING the nemesis owns the
        pairwise matrix: max_endpoints <= 65536, no drop() installed before, drop() refused while it is on"""
        nc = _lib.NemesisConfig(group, targets, interval_ns, self.now if start_ns is None else start_ns, time_limit_ns)
        return self._chk(self.L.ms_set_nemesis(self.h, C.byref(nc)))

    # journal -------------------------------------------------------------
    def journal_open(self, path):
        return self._chk(self.L.ms_journal_open(self.h, path.encode()))

    def journal_close(self):
        return self._chk(self.L.ms_journal_close(self.h))

    def drain(self, cap=1 << 20, bodies=True):
        """Everything journaled since the last call (including events stashed by run()); (events, bodies)."""
        parts = self._stash + [self._drain_now(cap, bodies)]
        self._stash = []
        ev = np.concatenate([p[0] for p in parts])
        bd = np.concatenate([p[1] for p in parts]) if bodies else None
        if getattr(self, "_jdecoder", None) is not None and len(ev):
            self._jdecoder.note(ev)          # the MS_JFMT_4 stream continues after these events
        return ev, bd

    def _drain_now(self, cap=1 << 20, bodies=True):
        evs, bds = [], []
        while True:
            ev = np.zeros(cap, dtype=EVENT_DTYPE)
            bd = np.zeros(cap, dtype=JBODY_DTYPE) if bodies else None
            n = C.c_size_t(0)
            self._chk(self.L.ms_journal_drain(self.h, ev.ctypes.data,
                                              bd.ctypes.data if bodies else None, cap, C.byref(n)))
            if n.value == 0:
                break
            evs.append(ev[:n.value])
            if bodies:
                bds.append(bd[:n.value])
        ev = np.concatenate(evs) if evs else np.zeros(0, dtype=EVENT_DTYPE)
        bd = (np.concatenate(bds) if bds else np.zeros(0, dtype=JBODY_DTYPE)) if bodies else None
        return ev, bd

    def run_streamed(self, until_ns, sink=None, fmt=_lib.JFMT_8, buf_events=0, decode=False, decoder=None):
        """ms_run_streamed: run to until_ns while the journal streams into pinned host memory.
        sink(batch_dict, rounds, events) is called per batch with numpy views that are only valid
        during the call (rounds: JROUND_DTYPE; events: u32 / u64 / 3 x u32 / EVENT_DTYPE by format);
        decode=True hands over EVENT_DTYPE records instead, expanded by ms_journal_decode or, for
        MS_JFMT_4, by `decoder` (a JournalDecoder that follows the stream; by default one kept with the Sim,
        which also hears about what drain() returns in between).
        Returns (events, bytes) streamed."""
        tot = [0, 0]
        err = []
        if decode and fmt == _lib.JFMT_4 and decoder is None:
            if getattr(self, "_jdecoder", None) is None:
                self._jdecoder = JournalDecoder()
            decoder = self._jdecoder

        def _cb(ctx, bp, rounds_p, events_p):
            try:
                b = bp.contents
                n = int(b.n_events)
                tot[0] += n
                tot[1] += n * int(b.format)
                if sink is not None:
                    rounds = np.ctypeslib.as_array(C.cast(rounds_p, C.POINTER(C.c_uint8)),
                                                   (int(b.n_rounds) * 32,)).view(_lib.JROUND_DTYPE)
                    if decode and decoder is not None:
                        ev = decoder.decode_raw(bp, rounds_p, events_p, n)
                    elif decode:
                        ev = np.zeros(n, dtype=EVENT_DTYPE)
                        self._chk(self.L.ms_journal_decode(bp, rounds_p, events_p, ev.ctypes.data))
                    else:
                        raw = np.ctypeslib.as_array(C.cast(events_p, C.POINTER(C.c_uint8)), (n * int(b.format),))
                        ev = (raw.view("<u4") if b.format == 4 else
                              raw.view("<u8") if b.format == 8 else raw.view("<u4").reshape(n, 3) if b.format == 12
                              else raw.view("<u8").reshape(n, 2) if b.format == 16 else raw.view(EVENT_DTYPE))
                    info = {k: int(getattr(b, k)) for k, _ in _lib.JBatch._fields_}
                    sink(info, rounds, ev)
                return 0
            except Exception as e:   # noqa: BLE001 -- must not propagate through the C frame
                err.append(e)
                return 1

        cb = _lib.JOURNAL_SINK(_cb)
        rc = self.L.ms_run_streamed(self.h, until_ns, fmt, buf_events, cb, None)
        if err:
            raise err[0]
        self._chk(rc)
        return tot[0], tot[1]

    def journal_written(self):
        return int(self.L.ms_journal_written(self.h))

    def stats(self):
        out = np.zeros(9, dtype=np.uint64)
        self._chk(self.L.ms_stats(self.h, out.ctypes.data))
        keys = ("send-count", "recv-count", "msg-count")
        return {cls: {k: int(out[i * 3 + j]) for j, k in enumerate(keys)}
                for i, cls in enumerate(("all", "clients", "servers"))}

    def counters(self):
        out = np.zeros(8, dtype=np.uint64)
        self._chk(self.L.ms_counters(self.h, out.ctypes.data))
        names = ("rounds", "sends", "recvs", "launches", "lost", "partition_drops", "max_window", "fallback_sorts")
        return {k: int(v) for k, v in zip(names, out)}

    RING_FIELDS = ("tail", "limit", "head", "ctail", "climit", "chead")

    def ring_counters(self):
        """ms_ring_counters: per-server uint32 arrays (index = server) of the 48-B inbox ring's tail / limit /
        head and the compact gossip ring's (ctail / climit / chead; zero without compact rings).  They wrap
        at 2^32: take differences modulo 2^32.  Servers of other shards read 0."""
        S = self.n_nodes
        out = np.zeros(6 * S, dtype=np.uint64)
        self._chk(self.L.ms_ring_counters(self.h, out.ctypes.data, out.size))
        return {k: out[i * S:(i + 1) * S].astype(np.uint32) for i, k in enumerate(self.RING_FIELDS)}

    def set_origin(self, round=0, msg_id=0, event_id=0, ring_pos=0, ring_stride=0):
        """ms_set_origin: start this fresh simulation as if `round` rounds, `msg_id` messages and `event_id`
        events had happened, with endpoint e's inbox counters at ring_pos + e * ring_stride (mod 2^32).
        For tests at the 32-bit boundaries of the engine's counters; only before any send, schedule or round."""
        return self._chk(self.L.ms_set_origin(self.h, round, msg_id, event_id, ring_pos & 0xFFFFFFFF,
                                              ring_stride & 0xFFFFFFFF))

    def timer_begin(self):
        return self._chk(self.L.ms_timer_begin(self.h))

    def timer_end(self):
        ms = C.c_double(0)
        self._chk(self.L.ms_timer_end(self.h, C.byref(ms)))
        return ms.value

    def profile(self, enable=True):
        return self._chk(self.L.ms_profile(self.h, 1 if enable else 0))

    def profile_read(self):
        ms = C.c_double(0)
        n = C.c_uint64(0)
        self._chk(self.L.ms_profile_read(self.h, C.byref(ms), C.byref(n)))
        return ms.value, int(n.value)

    def phase_cycles(self, enable=True):
        out = np.zeros(64, dtype=np.uint64)
        self._chk(self.L.ms_debug_phase_cycles(self.h, 1 if enable else 0, out.ctypes.data))
        return out.reshape(4, 16)

    def drain_into(self, ev_ptr, cap, body_ptr=None):
        """Drain up to `cap` events into caller memory (e.g. pinned); returns count."""
        n = C.c_size_t(0)
        self._chk(self.L.ms_journal_drain(self.h, ev_ptr, body_ptr, cap, C.byref(n)))
        return int(n.value)

    def node_set(self, node):
        n = self.L.ms_node_set(self.h, node, None, 0)
        out = np.zeros(max(n, 1), dtype=np.uint32)
        self.L.ms_node_set(self.h, node, out.ctypes.data, n)
        return out[:n]

    def client_replies(self):
        return int(self.L.ms_client_replies(self.h))

    def undeliverable(self):
        """Sends dropped because src / dest was not a registered endpoint (warning counter)."""
        return int(self.L.ms_undeliverable(self.h))

    RAFT_FIELDS = ("state", "term", "voted_for", "commit_index", "last_applied", "leader", "log_size", "kv_size")

    def raft_state(self, node):
        """RaftNode fields (demo/python/raft.py:196-221); state 0 nascent / 1 follower / 2 candidate /
        3 leader; voted_for and leader are -1 when unset."""
        out = np.zeros(8, dtype=np.uint64)
        self._chk(self.L.ms_raft_state(self.h, node, out.ctypes.data))
        d = dict(zip(self.RAFT_FIELDS, (int(x) for x in out)))
        d["voted_for"] -= 1
        d["leader"] -= 1
        return d

    PROXY_FIELDS = ("crashed", "next_msg_id", "pending")

    def proxy_state(self, node):
        """a lin-kv proxy's fields (ms_raft_state on MS_W_KV_PROXY): crashed 0 / 1, the last msg_id it sent, closures
        pending"""
        out = np.zeros(8, dtype=np.uint64)
        self._chk(self.L.ms_raft_state(self.h, node, out.ctypes.data))
        return dict(zip(self.PROXY_FIELDS, (int(x) for x in out[:3])))


HIST_TYPES = ("invoke", "ok", "fail", "info")              # MS_H_*
HF_KV_READ, HF_KV_WRITE, HF_KV_CAS = 2, 3, 4              # MS_HF_KV_*
HF_KAFKA_SEND, HF_KAFKA_POLL, HF_KAFKA_ASSIGN, HF_KAFKA_CRASH = 10, 11, 12, 13   # MS_HF_KAFKA_*
HF_COUNTER_ADD = 14                                       # MS_HF_COUNTER_ADD
HF_TXN_RW = 15                                            # MS_HF_TXN_RW
H_NEMESIS = 0xFFFFFFFF                                    # MS_H_NEMESIS: the client of a nemesis record
HF_NEM_ONE, HF_NEM_MAJORITY, HF_NEM_MINORITY_THIRD, HF_NEM_STOP = 5, 6, 7, 8   # MS_HF_NEM_*
HF_NEM_MAJORITIES_RING = 9                                # MS_HF_NEM_MAJORITIES_RING
NEM_ONE, NEM_MAJORITY, NEM_MINORITY_THIRD = 1, 2, 4       # ms_nemesis_config.targets bits
NEM_MAJORITIES_RING = 16


def nemesis_grudge(seed, cluster, g, op, target):
    """ms_nemesis_grudge: the grudge of a nemesis start record (op = its op, target = its f, cluster = its value) in a
    simulation with this seed and g servers per cluster; uint32 array, entry i for server cluster * g + i.  For
    HF_NEM_ONE / _MAJORITY / _MINORITY_THIRD it is 0 (side A) / 1 (side B); for HF_NEM_MAJORITIES_RING it is the
    server's ring position p, and the server at p receives from the one at q iff (q - p + h) % g < m, with
    m = g // 2 + 1 and h = m // 2"""
    out = np.zeros(max(g, 1), dtype=np.uint32)
    rc = _lib.lib().ms_nemesis_grudge(seed & 0xFFFFFFFF, seed >> 32, cluster, g, op, target, out.ctypes.data)
    if rc < 0:
        raise SimError(rc, _lib.lib().ms_last_error(None).decode())
    return out[:g]


def kv_history(records, first_client, group_clients):
    """The lin-kv clients' records (Sim.history() after add_kv_clients; first_client, group_clients =
    Sim.kv_groups) as the histories a register checker consumes: {(group, key): [op, ...]} in history order,
    one per register -- a group works on one cluster, so equal keys of different groups are different
    registers.  Each op is {"process", "type", "f", "value", "time", "error"} in Jepsen's shape for independent
    keys: value (k, v) for a read (v None unless it is an :ok) and a write, (k, (from, to)) for a cas;
    process = the client's endpoint index.  Nemesis records (client H_NEMESIS) are left out."""
    out = {}
    for r in records:
        if int(r["client"]) == H_NEMESIS:
            continue
        f, v = int(r["f"]), int(r["value"])
        k, a, b = v & 0xFFFF, (v >> 16) & 0xFF, v >> 24
        if f == HF_KV_READ:
            name, val = "read", (k, a if r["type"] == 1 else None)
        elif f == HF_KV_WRITE:
            name, val = "write", (k, a)
        elif f == HF_KV_CAS:
            name, val = "cas", (k, (a, b))
        else:
            raise ValueError("not a lin-kv history record: f = %d" % f)
        out.setdefault(((int(r["client"]) - first_client) // group_clients, k), []).append({"process": int(r["client"]), "type": HIST_TYPES[int(r["type"])], "f": name,
                                      "value": val, "time": int(r["time_ns"]), "error": int(r["error"]) or None})
    return out


def topology(name, n, node):
    out = np.zeros(max(n, 4), dtype=np.uint32)
    k = _lib.lib().ms_topology(TOPOLOGIES[name], n, node, out.ctypes.data, out.size)
    return out[:k].tolist()
