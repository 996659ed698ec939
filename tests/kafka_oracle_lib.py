"""TEST INFRASTRUCTURE: ctypes binding of tests/native/kafka_oracle.cpp, the oracle twin of the kafka workload
(MS_W_KAFKA): the CPU oracle plus the single-node kafka node and the kafka clients.  The library contains the whole
oracle, so a Sim made here is an oracle_lib.Sim in every other respect; its rounds, runs and receives are the kafka
twin's."""
import ctypes as C
import os
import subprocess

import numpy as np

import kv_oracle_lib as KV
import oracle_lib as O
from maelstrom_b200._lib import KAFKA_HIST_DTYPE

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "native", "kafka_oracle.cpp")
OUT = os.path.join(KV.OUT_DIR, "libkafka_oracle.so")
DEPS = [SRC, os.path.join(os.path.dirname(HERE), "oracle", "oracle.cpp"),
        os.path.join(os.path.dirname(HERE), "oracle", "oracle.h")]
W_KAFKA = 7                                               # MS_W_KAFKA
_lib = None


class KafkaConfig(C.Structure):                          # orkf_config = ms_kafka_gen_config
    _fields_ = [("n_clients", C.c_uint32), ("assign_permille", C.c_uint32), ("crash_permille", C.c_uint32),
                ("pad", C.c_uint32), ("interval_ns", C.c_int64), ("timeout_ns", C.c_int64), ("time_limit_ns", C.c_int64)]


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
        L.orkf_new.restype = C.c_void_p
        L.orkf_new.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
        L.orkf_free.argtypes = [C.c_void_p]
        L.orkf_add_clients.argtypes = [C.c_void_p, C.POINTER(KafkaConfig), C.c_uint32]
        L.orkf_run.argtypes = [C.c_void_p, C.c_int64]
        L.orkf_recv.argtypes = [C.c_void_p, C.c_uint32, C.c_int64, C.c_void_p]
        L.orkf_history.restype = C.c_size_t
        L.orkf_history.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
        L.orkf_log.restype = C.c_size_t
        L.orkf_log.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t]
        L.orkf_committed.restype = C.c_int64
        L.orkf_committed.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
        _lib = L
    return _lib


class Sim(O.Sim):
    """oracle_lib.Sim of n single-node kafka nodes with kafka_keys keys of kafka_log_cap messages"""

    def __init__(self, n_nodes, kafka_keys=0, kafka_log_cap=0, **kw):
        saved = O._lib
        try:
            O._lib = lib()
            O.Sim.__init__(self, n_nodes, workload=W_KAFKA, **kw)
        finally:
            O._lib = saved
        self.kf = self.L.orkf_new(self.h, kafka_keys, kafka_log_cap)

    def close(self):
        if getattr(self, "kf", None):
            self.L.orkf_free(self.kf)
            self.kf = None
        O.Sim.close(self)

    def add_kafka_clients(self, n_clients, interval_ns, time_limit_ns, assign_permille=0, crash_permille=0,
                          timeout_ns=0, first_name=0):
        kc = KafkaConfig(n_clients, assign_permille, crash_permille, 0, interval_ns, timeout_ns, time_limit_ns)
        return self._chk(self.L.orkf_add_clients(self.kf, C.byref(kc), first_name))

    def run(self, until_ns):
        return self._chk(self.L.orkf_run(self.kf, until_ns))

    def step(self, n=1):
        raise NotImplementedError("the kafka oracle runs by time")

    def recv(self, endpoint, timeout_ns=0):
        out = np.zeros(1, dtype=O.MSG_DTYPE)
        rc = self._chk(self.L.orkf_recv(self.kf, endpoint, timeout_ns, out.ctypes.data))
        return out[0] if rc == 1 else None

    def kafka_history(self):
        out = np.zeros(self.L.orkf_history(self.kf, None, 0), dtype=KAFKA_HIST_DTYPE)
        self.L.orkf_history(self.kf, out.ctypes.data, len(out))
        return out

    def kafka_log(self, node, key):
        n = self.L.orkf_log(self.kf, node, key, None, 0)
        out = np.zeros(n, dtype=np.uint32)
        self.L.orkf_log(self.kf, node, key, out.ctypes.data, n)
        return out

    def kafka_committed(self, node, key):
        c = self.L.orkf_committed(self.kf, node, key)
        return None if c == -1 else self._chk(c)
