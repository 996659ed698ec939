"""TEST INFRASTRUCTURE: ctypes binding of tests/native/txn_rw_oracle.cpp, the oracle twin of the txn-rw-register
workload (MS_W_TXN_RW): the CPU oracle plus the node of txn_rw_register_hat.clj and the txn clients.  The library
contains the whole oracle, so a Sim made here is an oracle_lib.Sim in every other respect; its rounds, runs and
receives are the txn-rw-register twin's."""
import ctypes as C
import os
import subprocess

import numpy as np

import kv_oracle_lib as KV
import oracle_lib as O
from maelstrom_b200._lib import TXN_RW_ENTRY_DTYPE, TXN_RW_HIST_DTYPE

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "native", "txn_rw_oracle.cpp")
OUT = os.path.join(KV.OUT_DIR, "libtxn_rw_oracle.so")
DEPS = [SRC, os.path.join(os.path.dirname(HERE), "oracle", "oracle.cpp"),
        os.path.join(os.path.dirname(HERE), "oracle", "oracle.h")]
W_TXN_RW = 10                                             # MS_W_TXN_RW
_lib = None


class TxnRwConfig(C.Structure):                          # orrw_config = ms_txn_rw_gen_config
    _fields_ = [("n_clients", C.c_uint32), ("min_len", C.c_uint32), ("max_len", C.c_uint32), ("key_count", C.c_uint32),
                ("interval_ns", C.c_int64), ("timeout_ns", C.c_int64), ("time_limit_ns", C.c_int64),
                ("key_period_ns", C.c_int64)]


def build():
    os.makedirs(KV.OUT_DIR, exist_ok=True)
    if os.path.exists(OUT) and all(os.path.getmtime(OUT) >= os.path.getmtime(d) for d in DEPS):
        return OUT
    tmp = OUT + ".tmp.%d" % os.getpid()
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", SRC, "-o", tmp])
    os.replace(tmp, OUT)
    return OUT


def lib():
    """the library, with oracle_lib's own prototypes on the oracle's entry points"""
    global _lib
    if _lib is None:
        saved = O._lib, O._SO
        try:
            O._lib, O._SO = None, build()
            L = O.lib()
        finally:
            O._lib, O._SO = saved
        L.orrw_new.restype = C.c_void_p
        L.orrw_new.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
        L.orrw_free.argtypes = [C.c_void_p]
        L.orrw_add_clients.argtypes = [C.c_void_p, C.POINTER(TxnRwConfig), C.c_uint32]
        L.orrw_run.argtypes = [C.c_void_p, C.c_int64]
        L.orrw_recv.argtypes = [C.c_void_p, C.c_uint32, C.c_int64, C.c_void_p]
        L.orrw_history.restype = C.c_size_t
        L.orrw_history.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
        L.orrw_log.restype = C.c_size_t
        L.orrw_log.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t]
        L.orrw_state.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                 C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


class Sim(O.Sim):
    """oracle_lib.Sim of n txn-rw-register nodes in blocks of raft_group servers (0 = all), with txn_rw_keys keys and
    logs of txn_rw_log_cap txns; the replication thread sleeps gset_interval_ms (the engine's default: 100)"""

    def __init__(self, n_nodes, txn_rw_keys=0, txn_rw_log_cap=0, gset_interval_ms=100, **kw):
        saved = O._lib
        try:
            O._lib = lib()
            O.Sim.__init__(self, n_nodes, workload=W_TXN_RW, gset_interval_ms=gset_interval_ms, **kw)
        finally:
            O._lib = saved
        self.rw = self.L.orrw_new(self.h, txn_rw_keys, txn_rw_log_cap)

    def close(self):
        if getattr(self, "rw", None):
            self.L.orrw_free(self.rw)
            self.rw = None
        O.Sim.close(self)

    def add_txn_rw_clients(self, n_clients, interval_ns, time_limit_ns, key_period_ns, key_count=1, min_len=1,
                           max_len=4, timeout_ns=0, first_name=0):
        rc = TxnRwConfig(n_clients, min_len, max_len, key_count, interval_ns, timeout_ns, time_limit_ns, key_period_ns)
        return self._chk(self.L.orrw_add_clients(self.rw, C.byref(rc), first_name))

    def run(self, until_ns):
        return self._chk(self.L.orrw_run(self.rw, until_ns))

    def step(self, n=1):
        raise NotImplementedError("the txn-rw-register oracle runs by time")

    def recv(self, endpoint, timeout_ns=0):
        out = np.zeros(1, dtype=O.MSG_DTYPE)
        rc = self._chk(self.L.orrw_recv(self.rw, endpoint, timeout_ns, out.ctypes.data))
        return out[0] if rc == 1 else None

    def txn_rw_history(self):
        out = np.zeros(self.L.orrw_history(self.rw, None, 0), dtype=TXN_RW_HIST_DTYPE)
        self.L.orrw_history(self.rw, out.ctypes.data, len(out))
        return out

    def txn_rw_log(self, node):
        out = np.zeros(self.L.orrw_log(self.rw, node, None, 0), dtype=TXN_RW_ENTRY_DTYPE)
        self.L.orrw_log(self.rw, node, out.ctypes.data, len(out))
        return out

    def _state(self, node):
        lamport, n, unrep, pend = C.c_uint64(0), C.c_uint32(0), C.c_uint32(0), C.c_uint32(0)
        k = self._chk(self.L.orrw_state(self.rw, node, C.byref(lamport), C.byref(n), None, None, 0, C.byref(unrep),
                                        C.byref(pend)))
        val, ts = np.zeros(k, dtype=np.uint32), np.zeros(k, dtype=np.uint64)
        self._chk(self.L.orrw_state(self.rw, node, C.byref(lamport), C.byref(n), val.ctypes.data, ts.ctypes.data, k,
                                    C.byref(unrep), C.byref(pend)))
        return (lamport.value, n.value, val, ts), (unrep.value, pend.value)

    def txn_rw_state(self, node):
        return self._state(node)[0]

    def unreplicated(self, node):
        """(size of the node's unreplicated map, the fewest nodes any of its txn+s still waits for)"""
        return self._state(node)[1]
