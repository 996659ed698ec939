"""TEST INFRASTRUCTURE: ctypes binding of tests/native/counter_oracle.cpp, the oracle twin of the g-counter and
pn-counter workloads (MS_W_G_COUNTER / MS_W_PN_COUNTER): the CPU oracle plus the PN-counter node and the counter
clients.  The library contains the whole oracle, so a Sim made here is an oracle_lib.Sim in every other respect (its
history() is the counter clients'); its rounds, runs and receives are the counter twin's."""
import ctypes as C
import os
import subprocess

import numpy as np

import kv_oracle_lib as KV
import oracle_lib as O

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "native", "counter_oracle.cpp")
OUT = os.path.join(KV.OUT_DIR, "libcounter_oracle.so")
DEPS = [SRC, os.path.join(os.path.dirname(HERE), "oracle", "oracle.cpp"),
        os.path.join(os.path.dirname(HERE), "oracle", "oracle.h")]
WORKLOADS = {"g-counter": 8, "pn-counter": 9}             # MS_W_G_COUNTER / MS_W_PN_COUNTER
_lib = None


class CounterConfig(C.Structure):                          # orct_config = ms_gen_config
    _fields_ = [("n_clients", C.c_uint32), ("read_permille", C.c_uint32), ("interval_ns", C.c_int64),
                ("timeout_ns", C.c_int64), ("time_limit_ns", C.c_int64), ("quiet_ns", C.c_int64)]


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
        L.orct_new.restype = C.c_void_p
        L.orct_new.argtypes = [C.c_void_p]
        L.orct_free.argtypes = [C.c_void_p]
        L.orct_add_clients.argtypes = [C.c_void_p, C.POINTER(CounterConfig), C.c_uint32]
        L.orct_run.argtypes = [C.c_void_p, C.c_int64]
        L.orct_recv.argtypes = [C.c_void_p, C.c_uint32, C.c_int64, C.c_void_p]
        L.orct_state.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t]
        _lib = L
    return _lib


class Sim(O.Sim):
    """oracle_lib.Sim of n counter nodes in blocks of raft_group servers (0 = all)"""

    def __init__(self, n_nodes, workload="pn-counter", **kw):
        saved = O._lib
        try:
            O._lib = lib()
            O.Sim.__init__(self, n_nodes, workload=WORKLOADS[workload], **kw)
        finally:
            O._lib = saved
        self.ct = self.L.orct_new(self.h)

    def close(self):
        if getattr(self, "ct", None):
            self.L.orct_free(self.ct)
            self.ct = None
        O.Sim.close(self)

    def add_gen_clients(self, n_clients, interval_ns, time_limit_ns, read_permille=None, timeout_ns=0, quiet_ns=0,
                        first_name=0):
        if read_permille is None:
            read_permille = 667 if self.workload == WORKLOADS["g-counter"] else 500
        gc = CounterConfig(n_clients, read_permille, interval_ns, timeout_ns, time_limit_ns, quiet_ns)
        return self._chk(self.L.orct_add_clients(self.ct, C.byref(gc), first_name))

    def run(self, until_ns):
        return self._chk(self.L.orct_run(self.ct, until_ns))

    def step(self, n=1):
        raise NotImplementedError("the counter oracle runs by time")

    def recv(self, endpoint, timeout_ns=0):
        out = np.zeros(1, dtype=O.MSG_DTYPE)
        rc = self._chk(self.L.orct_recv(self.ct, endpoint, timeout_ns, out.ctypes.data))
        return out[0] if rc == 1 else None

    def counter_state(self, node):
        n = self._chk(self.L.orct_state(self.ct, node, None, 0))
        out = np.zeros(n, dtype=np.int64)
        self.L.orct_state(self.ct, node, out.ctypes.data, n)
        return out[:n // 2], out[n // 2:]
