"""TEST INFRASTRUCTURE: ctypes binding of tests/native/kv_proxy_oracle.cpp, the oracle twin of the lin-kv proxy
(MS_W_KV_PROXY): the CPU oracle and the lin-kv clients' twin (tests/native/kv_oracle.cpp) plus the proxy node.  The
library contains the whole oracle, so a Sim made here is an oracle_lib.Sim in every other respect; its rounds, runs and
receives are the proxy twin's."""
import ctypes as C
import os
import subprocess

import numpy as np

import kv_oracle_lib as KV
import oracle_lib as O

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "native", "kv_proxy_oracle.cpp")
OUT = os.path.join(KV.OUT_DIR, "libkv_proxy_oracle.so")
DEPS = [SRC] + KV.DEPS
W_KV_PROXY = 6                                            # MS_W_KV_PROXY
PROXY_FIELDS = ("crashed", "next_msg_id", "pending")
_lib = None


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
        L.orkp_new.restype = C.c_void_p
        L.orkp_new.argtypes = [C.c_void_p, C.c_uint32]
        L.orkp_free.argtypes = [C.c_void_p]
        L.orkp_add_clients.argtypes = [C.c_void_p, C.POINTER(KV.KvConfig), C.c_uint32]
        L.orkp_run.argtypes = [C.c_void_p, C.c_int64]
        L.orkp_recv.argtypes = [C.c_void_p, C.c_uint32, C.c_int64, C.c_void_p]
        L.orkp_state.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
        _lib = L
    return _lib


class Sim(O.Sim):
    """oracle_lib.Sim of n lin-kv proxies over proxy_service ("lin-kv", "seq-kv", "lww-kv" or O.SVC's number)"""

    def __init__(self, n_nodes, proxy_service="lin-kv", **kw):
        svc = O.SVC[proxy_service] if isinstance(proxy_service, str) else int(proxy_service)
        saved = O._lib
        try:
            O._lib = lib()
            O.Sim.__init__(self, n_nodes, workload=W_KV_PROXY, **kw)
        finally:
            O._lib = saved
        self.kp = self.L.orkp_new(self.h, svc)
        if not self.kp:
            self.close()
            raise RuntimeError("kv proxy oracle: the backing service must be lin-kv, seq-kv or lww-kv")

    def close(self):
        if getattr(self, "kp", None):
            self.L.orkp_free(self.kp)
            self.kp = None
        O.Sim.close(self)

    def add_kv_clients(self, n_clients, interval_ns, time_limit_ns, key_period_ns, keys_per_group=1, value_range=0,
                       timeout_ns=0, first_name=0):
        kc = KV.KvConfig(n_clients, value_range, keys_per_group, interval_ns, timeout_ns, time_limit_ns, key_period_ns)
        return self._chk(self.L.orkp_add_clients(self.kp, C.byref(kc), first_name))

    def run(self, until_ns):
        return self._chk(self.L.orkp_run(self.kp, until_ns))

    def step(self, n=1):
        raise NotImplementedError("the kv proxy oracle runs by time")

    def recv(self, endpoint, timeout_ns=0):
        out = np.zeros(1, dtype=O.MSG_DTYPE)
        rc = self._chk(self.L.orkp_recv(self.kp, endpoint, timeout_ns, out.ctypes.data))
        return out[0] if rc == 1 else None

    def proxy_state(self, node):
        """as maelstrom_b200.Sim.proxy_state"""
        out = np.zeros(8, dtype=np.uint64)
        self._chk(self.L.orkp_state(self.kp, node, out.ctypes.data))
        return dict(zip(PROXY_FIELDS, (int(x) for x in out[:3])))
