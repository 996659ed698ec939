"""The round kernels where their CTAs interleave.

On the H100 a size class of k_round is a persistent grid of SMs x occupancy CTAs that take tickets of one round
at the same time: the ticket cursor with its prefetched next index, the `done` counter and the last ticket's
commit, the slot_open / round decision of a CTA that starts late, ring and journal-chunk claims, the timing
wheel's block claims and its "first publish wins" path, k_snapshot's class-list appends and the three-phase
commit's k_commit_a / k_commit_c blocks all run with several CTAs in flight.  The emulator runs the CTAs of a
launch one after another unless MS_EMUL_CTAS=<seed> (simt_ctas(seed) here) is on: then they run on a pool of
worker threads, 2 x MS_EMUL_SMS resident at once, and a seeded baton may park the running CTA at its start, at
a __syncthreads(), an atomic, a fence or a spin-wait and resume another one (tests/native/emul).

Every case compares with the oracle as test_counter_origins.run_case does: the level-2 journal field by field,
bodies, stats, now, round, node sets, the compact-ring accounting where the scenario qualifies and closed-loop
client histories.  The [emul] variants run under the mode with MS_EMUL_SMS=4 (class grids of four CTAs) and
three seeds; the [cuda] variants run each case once.  MS_CTA_SEEDS=a:b widens the seed range."""
import ctypes as C
import os

import pytest

import oracle_lib as O
import test_counter_origins as T
from scenarios import make_pair, random_broadcast_ops

pytestmark = pytest.mark.usefixtures("engine_backend")

SMS = 4


def seeds():
    a, b = (int(x) for x in os.environ.get("MS_CTA_SEEDS", "1:4").split(":"))
    return list(range(a, b))


SEEDS = seeds()


def emul_lib_handle():
    import emul_lib
    L = emul_lib.load()
    L.simt_ctas.argtypes = [C.c_longlong]
    L.simt_cta_counts.argtypes = [C.c_char_p, C.POINTER(C.c_ulonglong), C.POINTER(C.c_ulonglong)]
    return L


def cta_counts(L, kern):
    """(launches of `kern` in which two CTAs overlapped, baton passes from one of its CTAs in mid-flight)"""
    a, b = C.c_ulonglong(), C.c_ulonglong()
    L.simt_cta_counts(kern, C.byref(a), C.byref(b))
    return a.value, b.value


@pytest.fixture
def ctas(engine_backend, monkeypatch):
    """ctas(seed): on the emulator, concurrent CTAs with that seed and SMS multiprocessors for the rest of the test;
    on the GPU, which has them anyway, nothing"""
    L = emul_lib_handle() if engine_backend == "emul" else None

    def on(seed, each=False):
        # each: the case has one seed (not one per seed), so the GPU runs it too
        if engine_backend == "cuda":
            if seed != SEEDS[0] and not each:
                pytest.skip("the emulator's CTA seed; the GPU runs the case once")
            return None
        monkeypatch.setenv("MS_EMUL_SMS", str(SMS))
        L.simt_ctas(seed)
        L.simt_cta_counts_reset()
        return L
    yield on
    if L is not None:
        L.simt_ctas(int(os.environ.get("MS_EMUL_CTAS", "-1") or -1))


def overlapped(L, kern):
    if L is not None:
        n, passes = cta_counts(L, kern)
        assert n > 0 and passes > 0, (kern, n, passes)


# ------------------------------------------------------------------------------------------- counter-origin scenarios
@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("name", sorted(T.SCENARIOS))
def test_scenarios(ctas, name, seed):
    L = ctas(seed)
    T.run_case(T.SCENARIOS[name], None)
    overlapped(L, b"k_round")


BROADCAST = ("bcast_compact", "bcast_lat_const", "mixed_128", "mixed_512")


@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("kind", ["r15", "r31", "all"])
@pytest.mark.parametrize("name", BROADCAST)
def test_broadcast_round_origins(engine_backend, ctas, name, kind, seed):
    # slot_tag keeps 31 bits of the round and the per-ticket table tag 15: a late CTA's decision across both
    base = T.base_run(name, engine_backend)            # where the boundaries go; computed once, sequentially
    L = ctas(seed)
    origin = T.make_origin(kind, base)
    res = T.run_case(T.SCENARIOS[name], origin, probe="ring_pos" in origin)
    T.check_crossed(kind, origin, res, base)
    if T.SCENARIOS[name].compact == "eq":
        assert res["compact"] == base["compact"] > 0
    overlapped(L, b"k_round")


# ------------------------------------------------------------------------------------------- heavy windows
def mixed_case(k_g, k_f):
    from test_compact_gossip import mixed_window

    def make():
        g, o, scenario, _ = mixed_window(k_g, k_f, server_ring_cap=4096, server_max_window=2048)
        return g, o, scenario
    return T.Case(make, False, compact="eq", node_sets=5)


def heavy_flood(seen):
    # bursts into a 4 x 4 grid: windows of more than 512 messages from several senders, so sender blocks of size
    # classes 2 and 3 reach a window in whatever order their CTAs claimed ring space
    n = 16

    def make():
        g, o = make_pair(n, topology="grid", n_values=4096, ring_cap=4096, max_window=4096, journal_cap_log2=20,
                         max_endpoints=n + 8)

        def scenario(s, body):
            cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(4)]
            ops, _ = random_broadcast_ops(n, cs, n_ticks=2, per_tick=1200, seed=41)
            s.schedule(ops)
            s.run(12_000_000)
            if T.is_engine(s):
                seen["max_window"] = s.counters()["max_window"]
        return g, o, scenario
    return T.Case(make, False, compact="eq", node_sets=n)


@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("name", ["flood", "mixed_1000_1047"])
def test_heavy_windows(ctas, name, seed):
    L = ctas(seed)
    seen = {}
    T.run_case(heavy_flood(seen) if name == "flood" else mixed_case(1000, 1047), None)
    if name == "flood":
        assert seen["max_window"] > 512
    if L is not None:                    # k_round<2, *> / k_round<3, *>
        assert sum(cta_counts(L, k)[0] for k in (b"7k_roundILi2", b"7k_roundILi3")) > 0


# ------------------------------------------------------------------------------------------- timing wheel
def wheel_case():
    # 25 servers, constant latency 2: every round the CTAs of a class file gossip into the same new slot, and a
    # block's first record and the rest of it are often filed by different CTAs.  The pool holds 112 blocks of 16
    # records (calendar 16 x 16), a few more than the busiest two slots need: blocks that a lost publish race
    # kept, instead of handing back, run it dry within the run.
    n = 25

    def make():
        g, o = make_pair(n, topology="grid", latency_dist="constant", latency_mean_ms=2, n_values=2048,
                         ring_cap=1024, max_window=512, journal_cap_log2=20, max_endpoints=n + 8,
                         calendar_slots=16, calendar_cap=16)

        def scenario(s, body):
            cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(3)]
            ops, _ = random_broadcast_ops(n, cs, n_ticks=40, per_tick=8, seed=12)
            s.schedule(ops)
            s.run(120_000_000)
        return g, o, scenario
    return T.Case(make, False, node_sets=n)


@pytest.mark.parametrize("seed", SEEDS)
def test_timing_wheel_blocks(ctas, seed):
    L = ctas(seed)
    res = T.run_case(wheel_case(), None)
    assert res["stats"]["all"]["send-count"] > 5000
    overlapped(L, b"k_round")
    overlapped(L, b"k_release")


# ------------------------------------------------------------------------------------------- three-phase commit
def many_tickets(latency):
    # room for more than 16 384 tickets: the round is committed by k_commit_a / b / c; 1100 clients give k_snapshot
    # five CTAs and k_commit_a / k_commit_c two
    n = 25

    def make():
        g, o = make_pair(n, topology="grid", n_values=512, max_endpoints=17000, ring_cap=256, max_window=256,
                         latency_dist="constant", latency_mean_ms=latency, journal_cap_log2=18)

        def scenario(s, body):
            cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(1100)]
            ops, _ = random_broadcast_ops(n, cs[:3], n_ticks=12, per_tick=6, seed=4)
            s.schedule(ops)
            s.run((14 + 60 * latency) * 1_000_000)
        return g, o, scenario
    return T.Case(make, False, node_sets=n)


@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("latency", [0, 2])
def test_three_phase_commit(ctas, latency, seed):
    L = ctas(seed)
    res = T.run_case(many_tickets(latency), None)
    assert len(res["ev"]) > 3000
    for k in (b"k_snapshot", b"k_commit_a", b"k_commit_c"):
        overlapped(L, k)


# ------------------------------------------------------------------------------------------- streamed journal
@pytest.mark.parametrize("fmt", [4, 8, 12, 32])
def test_streamed_formats(ctas, fmt):
    # one seed per format (the flood is the file's slowest case): the four formats cover the three seeds
    from test_stream_overlap import Streamer, compare, flood_pair
    L = ctas(SEEDS[fmt % len(SEEDS)], each=True)
    g, o = flood_pair()
    s = Streamer(g, fmt, 1500)
    s.run(80_000_000)
    o.run(80_000_000)
    compare(s.journal(), o, g)
    g.close()
    overlapped(L, b"k_round")


@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("fmt", [8, 32])
def test_streamed_shards(engine_backend, ctas, fmt, seed):
    # a shard's k_journal_pack appends each chunk's events with one claim per chunk, from all of its CTAs
    if engine_backend == "cuda":
        pytest.skip("emulated shards: two GPUs are tests/test_gpu_sharded.py")
    import test_emul_sharded as S
    L = ctas(seed)
    S.test_emulated_shards_stream_their_journal(2, fmt, 0)
    overlapped(L, b"k_journal_pack")


# ------------------------------------------------------------------------------------------- emulated shards
@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("glue", [True, False], ids=["glue", "no_glue"])
def test_two_shards(engine_backend, ctas, monkeypatch, glue, seed):
    # every shard's host thread has its own pool and baton; gossip over the shard boundary claims peer rings
    if engine_backend == "cuda":
        pytest.skip("emulated shards: two GPUs are tests/test_gpu_sharded.py")
    import test_emul_sharded as S
    L = ctas(seed)
    S.test_emulated_shards_claim_peer_compact_rings(2, glue, monkeypatch)
    overlapped(L, b"k_round")


# ------------------------------------------------------------------------------------------- errors
@pytest.mark.parametrize("seed", SEEDS)
def test_capacity_errors(ctas, seed):
    # one receiver overflows, so what the latched error names does not depend on which CTA latched it first
    import test_compact_gossip as G
    ctas(seed)
    G.test_window_overflow_is_decided_by_the_sum()
    G.test_compact_ring_overflow_names_the_receiver()


@pytest.mark.parametrize("seed", SEEDS)
def test_first_of_several_errors(ctas, seed):
    # two receivers overflow their compact rings in the same round, claimed by CTAs of their own: the first CAS
    # latches one of them (DESIGN 3.6: which one may depend on the CTA order), and it stays latched
    import maelstrom_b200 as mb
    ctas(seed)
    g = mb.Sim(7, topology="line", n_values=256, ring_cap=1024, max_window=64, server_ring_cap=64)
    c = g.add_endpoint("c0", O.KIND_SIM_CLIENT)
    for v in range(120):                 # 1 and 3 overflow 2's ring, 3 and 5 overflow 4's
        g.send(c, (1, 3, 5)[v // 40], mb.body("broadcast", msg_id=v + 1, p0=v))
    g.step(1)
    with pytest.raises(mb.SimError) as e:
        g.step(1)
    msg = str(e.value)
    assert "inbox ring overflow" in msg and ("at endpoint 2 " in msg or "at endpoint 4 " in msg), msg
    r = g.round
    with pytest.raises(mb.SimError) as e2:
        g.step(1)
    assert str(e2.value) == msg and g.round == r
    g.close()


# ------------------------------------------------------------------------------------------- the mode itself
def test_mode_is_deterministic(engine_backend, ctas):
    # the same seed gives the same schedule: the same baton passes, kernel by kernel
    if engine_backend != "emul":
        pytest.skip("a property of the emulator")
    runs = []
    for seed in (SEEDS[0], SEEDS[0], SEEDS[0] + 1000):
        L = ctas(seed)
        T.run_case(T.SCENARIOS["bcast_lat_const"], None)
        runs.append([cta_counts(L, k) for k in (b"k_round", b"k_snapshot", b"k_release")])
    assert runs[0] == runs[1]
    assert runs[0][0][1] > 0
    assert runs[2] != runs[0]


def test_mode_off_runs_ctas_in_order(engine_backend, ctas):
    if engine_backend != "emul":
        pytest.skip("a property of the emulator")
    L = ctas(SEEDS[0])
    L.simt_ctas(-1)
    T.run_case(T.SCENARIOS["bcast_compact"], None)
    assert cta_counts(L, b"k_") == (0, 0)
