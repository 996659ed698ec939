"""TEST INFRASTRUCTURE: ctypes binding of tests/native/kv_oracle.cpp, the CPU oracle plus the twin of the engine's
closed-loop lin-kv clients (ms_add_kv_clients).  The library contains the whole oracle, so a Sim made here is an
oracle_lib.Sim in every other respect."""
import ctypes as C
import os
import subprocess

import oracle_lib as O

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "native", "kv_oracle.cpp")
OUT_DIR = os.path.join(HERE, "native", "_build")
OUT = os.path.join(OUT_DIR, "libkv_oracle.so")
DEPS = [SRC, os.path.join(ROOT, "oracle", "oracle.cpp"), os.path.join(ROOT, "oracle", "oracle.h"),
        os.path.join(ROOT, "maelstrom_b200", "csrc", "ms_tree.h")]
_lib = None


class KvConfig(C.Structure):    # orkv_config
    _fields_ = [("n_clients", C.c_uint32), ("value_range", C.c_uint32), ("keys_per_group", C.c_uint32),
                ("interval_ns", C.c_int64), ("timeout_ns", C.c_int64), ("time_limit_ns", C.c_int64),
                ("key_period_ns", C.c_int64)]


def build():
    os.makedirs(OUT_DIR, exist_ok=True)
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
        L.orkv_add_clients.restype = C.c_void_p
        L.orkv_add_clients.argtypes = [C.c_void_p, C.POINTER(KvConfig), C.c_uint32]
        L.orkv_free.argtypes = [C.c_void_p]
        L.orkv_first.restype = C.c_uint32
        L.orkv_first.argtypes = [C.c_void_p]
        L.orkv_run.argtypes = [C.c_void_p, C.c_int64]
        _lib = L
    return _lib


class Sim(O.Sim):
    """oracle_lib.Sim whose rounds, once add_kv_clients has been called, run the lin-kv clients too"""

    def __init__(self, *a, **kw):
        saved = O._lib
        try:
            O._lib = lib()
            O.Sim.__init__(self, *a, **kw)
        finally:
            O._lib = saved
        self.kv = None

    def close(self):
        if getattr(self, "kv", None):
            self.L.orkv_free(self.kv)
            self.kv = None
        O.Sim.close(self)

    def add_kv_clients(self, n_clients, interval_ns, time_limit_ns, key_period_ns, keys_per_group=1, value_range=0,
                       timeout_ns=0, first_name=0):
        if self.kv:
            raise RuntimeError("the lin-kv clients exist already")
        kc = KvConfig(n_clients, value_range, keys_per_group, interval_ns, timeout_ns, time_limit_ns, key_period_ns)
        self.kv = self.L.orkv_add_clients(self.h, C.byref(kc), first_name)
        if not self.kv:
            raise RuntimeError("kv oracle: bad configuration")
        return self.L.orkv_first(self.kv)

    def run(self, until_ns):
        if not self.kv:
            return O.Sim.run(self, until_ns)
        return self._chk(self.L.orkv_run(self.kv, until_ns))

    def step(self, n=1):
        if self.kv:
            raise NotImplementedError("the kv oracle runs by time")
        return O.Sim.step(self, n)
