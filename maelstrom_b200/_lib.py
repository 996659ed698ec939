"""ctypes loader for libmaelstrom_b200.so (built in-tree by __graft_entry__.build()).

Fails loudly when the library is missing: there is no CPU / PyTorch fallback.
"""
import ctypes as C
import os

import numpy as np

_DIR = os.path.dirname(os.path.abspath(__file__))
# MS_B200_LIB: another build of the same library (kernel tuning experiments), never a different implementation
SO_PATH = os.environ.get("MS_B200_LIB") or os.path.join(_DIR, "libmaelstrom_b200.so")

MSG_DTYPE = np.dtype([("id", "<u8"), ("deadline_ns", "<i8"), ("src", "<u4"), ("dest", "<u4"),
                      ("msg_id", "<u4"), ("in_reply_to", "<u4"), ("type", "<u2"), ("flags", "<u2"),
                      ("p0", "<u4"), ("p1", "<u8")])
EVENT_DTYPE = np.dtype([("event_id", "<u8"), ("time_ns", "<i8"), ("msg_id", "<u8"),
                        ("src", "<u4"), ("dest", "<u4")])
JBODY_DTYPE = np.dtype([("id", "<u8"), ("msg_id", "<u4"), ("in_reply_to", "<u4"), ("type", "<u2"),
                        ("flags", "<u2"), ("p0", "<u4"), ("p1", "<u8")])
BODY_DTYPE = np.dtype([("type", "<u2"), ("flags", "<u2"), ("msg_id", "<u4"), ("in_reply_to", "<u4"),
                       ("p0", "<u4"), ("p1", "<u8")])
OP_DTYPE = np.dtype([("time_ns", "<i8"), ("src", "<u4"), ("dest", "<u4"), ("body", BODY_DTYPE)])
assert MSG_DTYPE.itemsize == 48 and EVENT_DTYPE.itemsize == 32 and JBODY_DTYPE.itemsize == 32
assert BODY_DTYPE.itemsize == 24 and OP_DTYPE.itemsize == 40


class Config(C.Structure):
    _fields_ = [("n_nodes", C.c_uint32), ("workload", C.c_uint32), ("topology", C.c_uint32),
                ("latency_dist", C.c_uint32), ("latency_mean_ms", C.c_uint32),
                ("seed_lo", C.c_uint32), ("seed_hi", C.c_uint32), ("p_loss", C.c_double),
                ("n_values", C.c_uint32), ("gset_interval_ms", C.c_uint32),
                ("max_endpoints", C.c_uint32), ("ring_cap", C.c_uint32), ("max_window", C.c_uint32),
                ("journal_cap_log2", C.c_uint32), ("journal_level", C.c_uint32),
                ("journal_discard", C.c_uint32), ("calendar_slots", C.c_uint32),
                ("calendar_cap", C.c_uint32), ("mailbox_cap", C.c_uint32), ("inject_cap", C.c_uint32),
                ("device", C.c_int32), ("threads_per_node", C.c_uint32), ("n_shards", C.c_uint32),
                ("shard_id", C.c_uint32), ("reserved", C.c_uint32 * 6),
                ("server_ring_cap", C.c_uint32), ("server_max_window", C.c_uint32)]


class Body(C.Structure):
    _fields_ = [("type", C.c_uint16), ("flags", C.c_uint16), ("msg_id", C.c_uint32),
                ("in_reply_to", C.c_uint32), ("p0", C.c_uint32), ("p1", C.c_uint64)]


class GenConfig(C.Structure):   # ms_gen_config
    _fields_ = [("n_clients", C.c_uint32), ("read_permille", C.c_uint32), ("interval_ns", C.c_int64),
                ("timeout_ns", C.c_int64), ("time_limit_ns", C.c_int64), ("quiet_ns", C.c_int64)]


HIST_DTYPE = np.dtype([("time_ns", "<i8"), ("order", "<u8"), ("client", "<u4"), ("op", "<u4"), ("type", "u1"),
                       ("f", "u1"), ("error", "<u2"), ("value", "<u4")])
assert HIST_DTYPE.itemsize == 32


class JBatch(C.Structure):      # ms_jbatch
    _fields_ = [("first_event", C.c_uint64), ("n_events", C.c_uint64), ("n_rounds", C.c_uint64),
                ("now", C.c_int64), ("round", C.c_uint64), ("next_event", C.c_uint64),
                ("format", C.c_uint32), ("overflow", C.c_uint32), ("more", C.c_uint32), ("error", C.c_uint32),
                ("range_events", C.c_uint64)]


JROUND_DTYPE = np.dtype([("round", "<u8"), ("time_ns", "<i8"), ("ev_base", "<u8"), ("id_ref", "<u8")])
JOURNAL_SINK = C.CFUNCTYPE(C.c_int, C.c_void_p, C.POINTER(JBatch), C.c_void_p, C.c_void_p)
JFMT_EVENT, JFMT_12, JFMT_8, JFMT_16, JFMT_4 = 32, 12, 8, 16, 4

# every symbol include/maelstrom_b200.h declares: (restype, argtypes)
_P = C.c_void_p
SYMBOLS = {
    "ms_abi_version": (C.c_uint32, []),
    "ms_create": (_P, [C.POINTER(Config)]),
    "ms_destroy": (None, [_P]),
    "ms_last_error": (C.c_char_p, [_P]),
    "ms_start_nodes": (C.c_int, [_P, C.c_uint32]),
    "ms_stop_nodes": (C.c_int, [_P]),
    "ms_add_endpoint": (C.c_int, [_P, C.c_char_p, C.c_int]),
    "ms_remove_endpoint": (C.c_int, [_P, C.c_uint32]),
    "ms_endpoint_index": (C.c_int, [_P, C.c_char_p]),
    "ms_send": (C.c_int64, [_P, C.c_uint32, C.c_uint32, C.POINTER(Body)]),
    "ms_recv": (C.c_int, [_P, C.c_uint32, C.c_int64, _P]),
    "ms_send_json": (C.c_int64, [_P, C.c_char_p]),
    "ms_recv_json": (C.c_int, [_P, C.c_uint32, C.c_int64, C.c_char_p, C.c_size_t]),
    "ms_add_gen_clients": (C.c_int, [_P, _P, C.c_uint32]),
    "ms_history_drain": (C.c_int, [_P, _P, C.c_size_t, C.POINTER(C.c_size_t)]),
    "ms_schedule_ops": (C.c_int, [_P, _P, C.c_size_t]),
    "ms_step": (C.c_int, [_P, C.c_uint64]),
    "ms_run": (C.c_int, [_P, C.c_int64]),
    "ms_now": (C.c_int64, [_P]),
    "ms_round": (C.c_uint64, [_P]),
    "ms_net_drop": (C.c_int, [_P, C.c_uint32, C.c_uint32]),
    "ms_net_heal": (C.c_int, [_P]),
    "ms_net_slow": (C.c_int, [_P]),
    "ms_net_fast": (C.c_int, [_P]),
    "ms_net_flaky": (C.c_int, [_P]),
    "ms_net_set_loss": (C.c_int, [_P, C.c_double]),
    "ms_net_partition": (C.c_int, [_P, _P, C.c_size_t]),
    "ms_journal_open": (C.c_int, [_P, C.c_char_p]),
    "ms_journal_close": (C.c_int, [_P]),
    "ms_journal_drain": (C.c_int, [_P, _P, _P, C.c_size_t, C.POINTER(C.c_size_t)]),
    "ms_journal_written": (C.c_uint64, [_P]),
    "ms_run_streamed": (C.c_int, [_P, C.c_int64, C.c_int, C.c_size_t, JOURNAL_SINK, _P]),
    "ms_journal_decode": (C.c_int, [C.POINTER(JBatch), _P, _P, _P]),
    "ms_jdecoder_create": (_P, [C.c_uint32]),
    "ms_jdecoder_destroy": (None, [_P]),
    "ms_jdecoder_decode": (C.c_int, [_P, C.POINTER(JBatch), _P, _P, _P]),
    "ms_jdecoder_note": (C.c_int, [_P, _P, C.c_size_t]),
    "ms_jdecoder_error": (C.c_char_p, [_P]),
    "ms_stats": (C.c_int, [_P, _P]),
    "ms_node_set": (C.c_size_t, [_P, C.c_uint32, _P, C.c_size_t]),
    "ms_client_replies": (C.c_uint64, [_P]),
    "ms_undeliverable": (C.c_uint64, [_P]),
    "ms_raft_state": (C.c_int, [_P, C.c_uint32, _P]),
    "ms_counters": (C.c_int, [_P, _P]),
    "ms_ring_counters": (C.c_int, [_P, _P, C.c_uint32]),
    "ms_set_origin": (C.c_int, [_P, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint32]),
    "ms_timer_begin": (C.c_int, [_P]),
    "ms_timer_end": (C.c_int, [_P, C.POINTER(C.c_double)]),
    "ms_profile": (C.c_int, [_P, C.c_int]),
    "ms_profile_read": (C.c_int, [_P, C.POINTER(C.c_double), C.POINTER(C.c_uint64)]),
    "ms_shard_handles": (C.c_int, [_P, _P]),
    "ms_shard_connect": (C.c_int, [_P, C.c_uint32, _P]),
    "ms_set_barrier": (C.c_int, [_P, _P, _P]),
    "ms_stream": (_P, [_P]),
    "ms_shard_owner": (C.c_uint32, [C.c_uint32, C.c_uint32, C.c_uint32]),
    "ms_debug_phase_cycles": (C.c_int, [_P, C.c_int, _P]),
    "ms_topology": (C.c_size_t, [C.c_uint32, C.c_uint32, C.c_uint32, _P, C.c_size_t]),
}

SHARD_BLOB_BYTES = 512
BARRIER_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p)
_lib = None


def lib():
    """Load the CUDA engine.  Raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(SO_PATH):
            raise ImportError(
                "maelstrom_b200: %s is missing -- run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a). There is no CPU fallback." % SO_PATH)
        L = C.CDLL(SO_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(L, name)   # AttributeError if the ABI is incomplete
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib
