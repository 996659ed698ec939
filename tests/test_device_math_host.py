"""CPU checks of the engine's own pure helpers (csrc/ms_device.cuh compiled for the host with
g++): Philox4x32-10 known answers, the integer-only exponential/uniform/constant latency draw
and the shard-ownership function, each against the published vectors and the oracle."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import oracle_lib as O

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def dm(tmp_path_factory):
    out = tmp_path_factory.mktemp("dm") / "libdevice_math_host.so"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", str(out),
                           os.path.join(HERE, "native", "device_math_host.cpp")])
    L = C.CDLL(str(out))
    L.dm_neg_log2_q32.restype = C.c_uint64
    L.dm_neg_log2_q32.argtypes = [C.c_uint64]
    L.dm_latency.restype = C.c_uint64
    L.dm_latency.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64, C.c_void_p]
    L.dm_owner.restype = C.c_uint32
    L.dm_owner.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32]
    L.dm_compact_round.restype = C.c_uint64
    L.dm_compact_round.argtypes = [C.c_uint64, C.c_uint32]
    return L


def philox(L, ctr, key):
    c = np.asarray(ctr, dtype=np.uint32)
    k = np.asarray(key, dtype=np.uint32)
    o = np.zeros(4, dtype=np.uint32)
    L.dm_philox(c.ctypes.data, k.ctypes.data, o.ctypes.data)
    return o.tolist()


def test_engine_philox_known_answers(dm):
    assert philox(dm, [0, 0, 0, 0], [0, 0]) == [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]
    assert philox(dm, [0xffffffff] * 4, [0xffffffff] * 2) == [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]
    assert philox(dm, [0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], [0xa4093822, 0x299f31d0]) == \
        [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1]
    rng = np.random.default_rng(3)
    for _ in range(200):
        ctr = rng.integers(0, 2 ** 32, 4).tolist()
        key = rng.integers(0, 2 ** 32, 2).tolist()
        assert philox(dm, ctr, key) == O.philox(ctr, key)


def test_engine_latency_draws_equal_oracle(dm):
    rng = np.random.default_rng(5)
    xs = rng.integers(0, 2 ** 32, size=(3000, 4), dtype=np.uint64).astype(np.uint32)
    for dist_name, dist in (("constant", 0), ("uniform", 1), ("exponential", 2)):
        for mean, scale in ((1, 1), (5, 1), (100, 1), (100, 10), (7, 100)):
            coeff = int(round(mean * scale * math.log(2.0) * 2 ** 32))
            # the host side computes the coefficient with llround(double) exactly like this
            for x in xs[:600]:
                got = dm.dm_latency(dist, mean, scale, coeff, x.ctypes.data)
                assert got == O.latency_draw(dist_name, mean, scale, x), (dist_name, mean, scale, x)
    # exact fixed-point identities of -log2(u), u = (X+1)/2^64
    assert dm.dm_neg_log2_q32(2 ** 64 - 1) == 0
    assert dm.dm_neg_log2_q32(2 ** 63 - 1) == 1 << 32            # u = 1/2
    assert dm.dm_neg_log2_q32(0) == 64 << 32                     # u = 2^-64


def test_engine_owner_function(dm):
    from maelstrom_b200.sharded import shard_owner
    for n_servers, extra in ((4096, 64), (25, 3), (7, 9)):
        for g in (1, 2, 3, 4, 8):
            owners = [dm.dm_owner(e, n_servers, g) for e in range(n_servers + extra)]
            assert owners == [shard_owner(e, n_servers, g) for e in range(n_servers + extra)]
            assert owners[:n_servers] == sorted(owners[:n_servers]) and max(owners) == (g - 1 if n_servers >= g else max(owners))
            counts = np.bincount(owners[:n_servers], minlength=g)
            assert counts.max() - counts.min() <= 1


def test_compact_round_rebuilds_the_sender_round(dm):
    # a compact gossip record keeps the low 32 bits of its sender's round; the receiver (at round R, the sender's
    # round + d) rebuilds the 64-bit round.  No simulation reaches round 2^32, so this is the only check there.
    rng = np.random.default_rng(11)
    receivers = [r for c in (2 ** 32, 2 ** 33, 5 * 2 ** 32) for r in range(c - 4, c + 5)]
    receivers += [int(x) for x in rng.integers(0, 2 ** 40, 200)] + [0, 1, 2 ** 40 - 1]
    for R in receivers:
        for d in (0, 1, 2, 3, 7, 64, 2 ** 16, 2 ** 31, 2 ** 32 - 1):
            s = R - d
            if s < 0:
                continue
            assert dm.dm_compact_round(R, s & 0xFFFFFFFF) == s, (R, d)
    # the newest round with those low bits that is not after R: never a later round, never 2^32 too early
    for R in (2 ** 32 - 1, 2 ** 32, 2 ** 32 + 1):
        for lo in (0, 1, 0xFFFFFFFE, 0xFFFFFFFF, R & 0xFFFFFFFF):
            got = dm.dm_compact_round(R, lo)
            assert got <= R and R - got < 2 ** 32 and got & 0xFFFFFFFF == lo, (R, lo, got)


def test_compact_order_key_is_monotone_across_2_32(dm):
    # k_round orders a window by (round << 24) | ticket with the round a compact slot rebuilds: consecutive
    # sender rounds across the 2^32 boundary (each read one round later) must give increasing keys
    for c in (2 ** 32, 2 ** 33, 2 ** 39):
        keys = []
        for s in range(c - 3, c + 4):
            rebuilt = dm.dm_compact_round(s + 1, s & 0xFFFFFFFF)
            assert rebuilt == s
            for ticket in (8, 9, 0xFFFFFF):
                keys.append(((rebuilt << 24) | ticket) & (2 ** 64 - 1))
        assert keys == sorted(keys) and len(set(keys)) == len(keys)
        assert keys[-1] == ((c + 3) << 24) | 0xFFFFFF          # no bit of the round lost to the 64-bit key


def test_bench_numpy_philox_matches_oracle():
    import bench
    got = bench.philox_u32(257, 1, offset=1000)
    want = [O.philox([1000 + i, 0, 0, 0], [bench.SEED & 0xFFFFFFFF, 1])[0] for i in range(257)]
    assert got.tolist() == want
