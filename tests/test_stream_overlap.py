"""ms_run_streamed where the journal stream overlaps the next batch's rounds.

The journal of batch i is planned, packed and copied out on its own stream while the rounds of batch i+1 run and
commit on the engine's stream.  Whatever the journal stream reads must therefore be fixed in stream order (the
mark k_stream_mark takes behind each batch's rounds) or belong to rounds that stay put until drained.  Every case
compares the streamed journal with the oracle's event for event, checks each batch header with a sink of its
own, and asserts stats, now and round.  The [emul] variants run under the emulator's asynchronous streams
(MS_EMUL_STREAMS, tests/native/emul), where the journal stream really runs while a round kernel is parked half
way; the [cuda] variants run on the GPU, once each, and add the bench topology and bench's own e2e configuration.

The pinned buffers the sink sees are the engine's, so they cannot be pre-filled with a sentinel; the event for
event comparison is what catches stale staging bytes."""
import argparse
import ctypes as C
import os

import numpy as np
import pytest

import oracle_lib as O
from scenarios import make_pair, random_broadcast_ops

pytestmark = pytest.mark.usefixtures("engine_backend")
cuda_only = pytest.mark.gpu

SEEDS = (11, 12, 13)
FIELDS = ("event_id", "time_ns", "msg_id", "src", "dest")


def emul_lib_handle():
    import emul_lib
    L = emul_lib.load()
    L.simt_streams.argtypes = [C.c_longlong]
    L.simt_interleaved.restype = C.c_ulonglong
    L.simt_interleaved.argtypes = [C.c_char_p, C.c_char_p]
    return L


@pytest.fixture
def overlap(engine_backend):
    """overlap(seed): on the emulator, asynchronous streams with that seed for the rest of the test"""
    L = emul_lib_handle() if engine_backend == "emul" else None

    def on(seed):
        if L is not None:
            L.simt_streams(seed)
            L.simt_interleaved_reset()
        return L
    yield on
    if L is not None:
        L.simt_streams(-1)


def only_first_seed_on_gpu(engine_backend, seed):
    # on the GPU the seed means nothing: run each case once
    if engine_backend == "cuda" and seed != SEEDS[0]:
        pytest.skip("the emulator's stream seed; the GPU runs the case once")


# ------------------------------------------------------------------------------------------- streaming
class Streamer:
    """Wraps an engine so that run(until) streams (ms_run_streamed) and every batch is checked; the journal is the
    streamed batches plus whatever drain() returned in between, in order."""

    def __init__(self, g, fmt, buf_events, drain_between=False, decoder=None):
        self.g, self.fmt, self.buf_events = g, fmt, buf_events
        self.drain_between = drain_between
        self.decoder = decoder
        self.parts = []
        self.n = 0                     # events handed over so far (streamed or drained)
        self.batches = []              # (first_event, n_events, n_rounds)
        self.max_round_events = 0

    def __getattr__(self, name):
        return getattr(self.g, name)

    def sink(self, info, rounds, ev):
        first, n = info["first_event"], info["n_events"]
        assert info["format"] == self.fmt and len(ev) == n <= self.buf_events
        assert first == self.n, ("batches are not contiguous", first, self.n)
        assert n <= info["next_event"] - first
        assert len(rounds) == info["n_rounds"] >= 1
        eb = rounds["ev_base"].astype(np.int64)
        assert eb[0] <= first and eb[-1] <= first + n                   # rows lie within the batch (a cut one may end on idle rounds)
        assert np.all(np.diff(rounds["round"].astype(np.int64)) == 1)
        assert np.all(np.diff(eb) >= 0)
        held = np.append(eb[1:], first + n) > np.maximum(eb, first)   # rows that hold events of this batch
        assert np.all(np.diff(eb[held]) > 0)
        if len(eb) > 1:
            self.max_round_events = max(self.max_round_events, int(np.diff(eb).max()))
        ids = ev["event_id"] & np.uint64((1 << 63) - 1)
        assert np.array_equal(ids, np.arange(first, first + n, dtype=np.uint64))
        self.parts.append(ev.copy())
        self.n += n
        self.batches.append((first, n, int(info["n_rounds"])))

    def drain_now(self):
        ev, _ = self.g.drain(bodies=False)
        if len(ev):
            assert int(ev["event_id"][0] & np.uint64((1 << 63) - 1)) == self.n
            self.parts.append(ev)
            self.n += len(ev)

    def run(self, until_ns):
        if self.drain_between:
            self.drain_now()
        self.g.run_streamed(until_ns, self.sink, fmt=self.fmt, buf_events=self.buf_events, decode=True,
                            decoder=self.decoder)
        return 0

    def journal(self):
        self.drain_now()
        return np.concatenate(self.parts) if self.parts else np.zeros(0, dtype=self.parts_dtype())

    def parts_dtype(self):
        from maelstrom_b200.engine import EVENT_DTYPE
        return EVENT_DTYPE


def compare(ev_g, o, g):
    ev_o, _ = o.journal()
    assert len(ev_g) == len(ev_o), (len(ev_g), len(ev_o))
    for f in FIELDS:
        if not np.array_equal(ev_g[f], ev_o[f]):
            bad = int(np.nonzero(ev_g[f] != ev_o[f])[0][0])
            raise AssertionError("streamed journal field %s differs first at event %d: engine=%s oracle=%s" %
                                 (f, bad, ev_g[bad], ev_o[bad]))
    assert g.stats() == o.stats() and g.now == o.now and g.round == o.round
    return ev_o


def flood_pair(n=36, jcap=11, per_tick=30, ticks=20, latency=0, **kw):
    """A broadcast flood whose largest round writes just under half of the 2^jcap-record raw ring: the most a round
    may write without ever overflowing while the stream lags (a round starts with up to half the ring undrained).
    A round that wrote more could overflow legitimately."""
    g, o = make_pair(n, topology="grid", n_values=8192, ring_cap=1024, max_window=512, journal_cap_log2=jcap,
                     journal_level=1, latency_dist="constant", latency_mean_ms=latency, **kw)
    cs = [g.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(4)]
    assert cs == [o.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(4)]
    ops, _ = random_broadcast_ops(n, cs, n_ticks=ticks, per_tick=per_tick, seed=31)
    g.schedule(ops)
    o.schedule(ops)
    return g, o


# ------------------------------------------------------------------------------------------- the emulator mode
def test_streams_mode_interleaves_the_journal_stream_with_rounds(engine_backend, overlap):
    # the self-test of MS_EMUL_STREAMS: some batch's plan, pack and finish run while a round kernel is parked
    if engine_backend != "emul":
        pytest.skip("a property of the emulator")
    L = overlap(SEEDS[0])
    g, o = flood_pair()
    s = Streamer(g, 8, 1 << 16)
    s.run(80_000_000)
    o.run(80_000_000)
    compare(s.journal(), o, g)
    for k in (b"k_stream_plan", b"k_journal_pack", b"k_stream_finish"):
        assert L.simt_interleaved(b"k_round", k) > 0, k
    g.close()


# ------------------------------------------------------------------------------------------- formats, batches
@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("fmt,buf_events", [(4, 1 << 16), (8, 1 << 16), (12, 1 << 16), (32, 1 << 16),
                                            (4, 733), (8, 300), (12, 1500), (32, 257)])
def test_formats_and_batch_sizes(engine_backend, overlap, fmt, buf_events, seed):
    # small buffers cut batches inside rounds and inside one ticket's chunk (a flood round is a few tickets of
    # hundreds of events each); the largest round writes just under half of the raw ring
    only_first_seed_on_gpu(engine_backend, seed)
    overlap(seed)
    g, o = flood_pair()
    s = Streamer(g, fmt, buf_events)
    s.run(80_000_000)
    o.run(80_000_000)
    compare(s.journal(), o, g)
    assert (1 << 11) // 4 < s.max_round_events <= (1 << 11) // 2
    if buf_events < 2000:
        assert any(n == buf_events for _, n, _ in s.batches)            # cut by the buffer
    g.close()


@pytest.mark.parametrize("batch_rounds", [1, 8, 32])
def test_batch_rounds(engine_backend, overlap, monkeypatch, batch_rounds):
    monkeypatch.setenv("MS_STREAM_BATCH_ROUNDS", str(batch_rounds))
    overlap(SEEDS[batch_rounds % 3])
    g, o = flood_pair()
    s = Streamer(g, 4, 900)
    s.run(9_000_000)
    s.run(80_000_000)
    o.run(80_000_000)
    compare(s.journal(), o, g)
    g.close()


def test_rows_table_cut(engine_backend, overlap, monkeypatch):
    # a batch whose events span more than kStreamRows (4096) rounds is cut at a round boundary: events, then 5 s of
    # idle rounds, then events again, with long batches and a buffer that keeps the stream behind the rounds
    monkeypatch.setenv("MS_STREAM_BATCH_ROUNDS", "1024")
    overlap(SEEDS[1])
    n = 9
    g, o = make_pair(n, topology="grid", n_values=4096, ring_cap=512, max_window=256, journal_cap_log2=16,
                     journal_level=1, history_rounds=16384)
    cs = [g.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(2)]
    assert cs == [o.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(2)]
    a, _ = random_broadcast_ops(n, cs, n_ticks=3, per_tick=20, seed=4)
    b, _ = random_broadcast_ops(n, cs, n_ticks=3, per_tick=20, seed=5)
    b["time_ns"] += 5000 * 1_000_000
    b["body"]["msg_id"] += 1000
    b["body"]["p0"] += 1000
    ops = np.concatenate([a, b])
    g.schedule(ops)
    o.schedule(ops)
    s = Streamer(g, 12, 64)
    s.run(5010 * 1_000_000)
    o.run(5010 * 1_000_000)
    compare(s.journal(), o, g)
    assert max(r for _, _, r in s.batches) == 4096
    g.close()


# ------------------------------------------------------------------------------------------- traffic shapes
def exp_latency_laps():
    # exponential latency on a 16-slot timing wheel, slowed twice: many messages lap the wheel
    def make():
        g, o = make_pair(16, topology="grid", latency_dist="exponential", latency_mean_ms=4, n_values=1024,
                         ring_cap=1024, max_window=512, journal_cap_log2=12, max_endpoints=24, calendar_slots=16,
                         calendar_cap=8192)

        def scenario(s, body):
            cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(3)]
            ops, _ = random_broadcast_ops(16, cs, n_ticks=8, per_tick=12, seed=6)
            s.schedule(ops)
            s.slow()
            s.slow()
            s.run(30_000_000)
            s.fast()
            s.run(400_000_000)
        return g, o, scenario
    return make


def origin_case(name):
    def make():
        import test_counter_origins as T
        return T.SCENARIOS[name].make()
    return make


def history_stretches():
    # closed-loop clients, the history drained between streamed stretches
    n, k = 9, 6

    def make():
        g, o = make_pair(n, topology="grid", n_values=1 << 12, ring_cap=1024, max_window=512, journal_cap_log2=12,
                         max_endpoints=n + 8)

        def scenario(s, body):
            s.add_gen_clients(k, interval_ns=2_000_000, time_limit_ns=40_000_000, read_permille=400,
                              timeout_ns=15_000_000, quiet_ns=20_000_000)
            hist = []
            for t in (10, 25, 45, 70):
                s.run(t * 1_000_000)
                h = s.history()
                hist += [tuple(int(r[f]) for f in ("time_ns", "order", "client", "op", "type", "f", "error", "value"))
                         for r in h]
            assert hist
            return hist
        return g, o, scenario
    return make


SHAPES = {
    "exp_laps": exp_latency_laps(),
    "loss": origin_case("loss"),
    "flaky": origin_case("flaky"),
    "partition": origin_case("partition"),
    "remove_readd": origin_case("remove_readd"),
    "gset": origin_case("gset"),
    "services": origin_case("services"),
    "txn": origin_case("txn"),
    "raft": origin_case("raft"),
    "gen_clients": history_stretches(),
}


@pytest.mark.parametrize("shape", sorted(SHAPES))
@pytest.mark.parametrize("fmt", [4, 32])
def test_traffic_shapes(engine_backend, overlap, shape, fmt):
    overlap(SEEDS[(sorted(SHAPES).index(shape) + fmt) % 3])
    g, o, scenario = SHAPES[shape]()
    s = Streamer(g, fmt, 501 if fmt == 4 else 3000)
    rg = scenario(s, __import__("maelstrom_b200").body)
    ro = scenario(o, O.body)
    assert rg == ro
    compare(s.journal(), o, g)
    g.close()


# ------------------------------------------------------------------------------------------- stopping, resuming
@pytest.mark.parametrize("fmt", [4, 8, 12, 32])
def test_streamed_stretches_between_run_and_drain(engine_backend, overlap, fmt):
    overlap(SEEDS[fmt % 3])
    g, o = flood_pair(latency=2, jcap=16)         # with latency a round can write more than half of 2^11
    s = Streamer(g, fmt, 1000, drain_between=True)
    for t in (5, 9, 17, 30):
        s.run(t * 1_000_000)
        g.run((t + 2) * 1_000_000)                 # ordinary running in between: run() drains what it must
    s.run(120_000_000)
    o.run(120_000_000)
    compare(s.journal(), o, g)
    g.close()


def test_format4_with_a_fresh_decoder_after_a_drain(engine_backend, overlap):
    # a decoder created after a full drain, with nothing in flight across the cut, follows the stream from there
    from maelstrom_b200.engine import JournalDecoder
    overlap(SEEDS[2])
    g, o = flood_pair(latency=0, ticks=6)
    s = Streamer(g, 4, 1000)
    s.run(3_000_000)
    g.run(40_000_000)                              # the flood is over: no message in flight
    s.drain_now()
    more, _ = random_broadcast_ops(36, list(range(36, 40)), n_ticks=4, per_tick=20, seed=9)
    more["time_ns"] += 45_000_000
    more["body"]["msg_id"] += 1000
    more["body"]["p0"] += 1000
    g.schedule(more)
    o.schedule(more)
    s.decoder = JournalDecoder(log2_window=22)
    s.run(60_000_000)
    o.run(60_000_000)
    compare(s.journal(), o, g)
    g.close()


def test_format4_decoder_window_too_small(engine_backend, overlap):
    # a :recv names its :send by id; a decoder whose window is smaller than the distance in flight cannot, and says so
    import maelstrom_b200 as mb
    from maelstrom_b200.engine import JournalDecoder
    overlap(SEEDS[0])
    g, _ = flood_pair(latency=3)
    with pytest.raises(mb.SimError) as e:
        g.run_streamed(60_000_000, lambda *a: None, fmt=4, decode=True, decoder=JournalDecoder(log2_window=6))
    assert "ms_jdecoder" in str(e.value)
    g.close()


# ------------------------------------------------------------------------------------------- GPU: bench scale
BENCH_N, BENCH_V, BENCH_TICKS = 4096, 1280, 2


def bench_topology_pair():
    from test_gpu_parity import hot_broadcast_ops
    n = BENCH_N
    g, o = make_pair(n, topology="grid", n_values=BENCH_V * BENCH_TICKS + 8, max_endpoints=n + 8, ring_cap=8192,
                     max_window=4096, journal_cap_log2=22, journal_level=1)
    cs = [g.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(4)]
    assert cs == [o.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(4)]
    ops = hot_broadcast_ops(n, cs, BENCH_TICKS, BENCH_V, [10 * 64 + 10, 11 * 64 + 11, 40 * 64 + 50], 900, seed=77)
    g.schedule(ops)
    o.schedule(ops)
    return g, o


@pytest.fixture(scope="module")
def bench_topology_oracle():
    _, o = bench_topology_pair()
    o.run(BENCH_TICKS * 1_000_000)
    ev_o, _ = o.journal()
    return ev_o, o.stats(), o.now, o.round


@cuda_only
@pytest.mark.parametrize("fmt", [4, 8, 12, 32])
def test_bench_topology_streamed(engine_backend, bench_topology_oracle, fmt):
    # 4096 nodes, 30.8 M messages, windows up to 2342, streamed through a 2^22-record raw ring: the stream keeps
    # the simulation behind it all the way (61.6 M events through a ring of 4.2 M)
    if engine_backend != "cuda":
        pytest.skip("61 M journal events: GPU only")
    ev_o, stats_o, now_o, round_o = bench_topology_oracle
    g, _ = bench_topology_pair()
    s = Streamer(g, fmt, 1 << 22)
    s.run(BENCH_TICKS * 1_000_000)
    ev_g = s.journal()
    assert len(ev_g) == len(ev_o) == 2 * BENCH_TICKS * BENCH_V * 12035
    for f in FIELDS:
        if not np.array_equal(ev_g[f], ev_o[f]):
            bad = int(np.nonzero(ev_g[f] != ev_o[f])[0][0])
            raise AssertionError("field %s differs first at event %d: engine=%s oracle=%s (batches around it: %s)" % (
                f, bad, ev_g[bad], ev_o[bad], [b for b in s.batches if b[0] <= bad < b[0] + b[1]]))
    assert g.stats() == stats_o and g.now == now_o and g.round == round_o
    assert s.max_round_events > (1 << 22) // 8           # rounds are a sizeable part of the ring
    assert g.counters()["max_window"] == 2342
    g.close()


_MIX = (np.uint64(0x9E3779B97F4A7C15), np.uint64(0xBF58476D1CE4E5B9), np.uint64(0x94D049BB133111EB),
        np.uint64(0xD6E8FEB86659FD93), np.uint64(0xA0761D6478BD642F))


def fold(ev):
    """order-independent digest of journal events: the sum of a 64-bit mix of the five fields of each"""
    with np.errstate(over="ignore"):
        h = (ev["event_id"].astype(np.uint64) * _MIX[0]) ^ (ev["time_ns"].astype(np.uint64) * _MIX[1])
        h ^= ev["msg_id"].astype(np.uint64) * _MIX[2]
        h ^= ((ev["src"].astype(np.uint64) << np.uint64(32)) | ev["dest"].astype(np.uint64)) * _MIX[3]
        h ^= h >> np.uint64(31)
        h *= _MIX[4]
        h ^= h >> np.uint64(29)
        return int(h.sum(dtype=np.uint64))


class Digest:
    def __init__(self):
        self.n = 0
        self.sum = 0
        self.lo, self.hi = None, None

    def add(self, ev):
        if not len(ev):
            return
        ids = ev["event_id"] & np.uint64((1 << 63) - 1)
        assert int(ids[0]) == self.n and int(ids[-1]) == self.n + len(ev) - 1       # in order, no gap
        self.n += len(ev)
        self.sum = (self.sum + fold(ev)) & ((1 << 64) - 1)


@cuda_only
def test_bench_e2e_configuration_streamed(engine_backend):
    # bench.py's e2e arm, two steps: its broadcast workload and ops, streamed as it streams them (MS_JFMT_4, its
    # default buffer), against the same steps read through ms_journal_drain in pieces
    if engine_backend != "cuda":
        pytest.skip("788 M events per step: GPU only")
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import bench
    import maelstrom_b200 as mb
    from maelstrom_b200 import _lib
    from maelstrom_b200.engine import EVENT_DTYPE, F_MSG_ID, F_APPENDS, OP_DTYPE, TYPES, JournalDecoder
    args = argparse.Namespace(config="broadcast", latency_ms=0, values_per_tick=0, ring_cap=8192, max_window=4096,
                              threads=0, journal_cap_log2=28, stream_events=1 << 26)
    wl = bench.make_workload(args)
    steps = 2
    step_ns = wl.step_ticks * bench.TICK_NS
    flags = {"msg_id": F_MSG_ID, "appends": F_APPENDS}

    def make():
        sim, c0 = bench.make_sim(mb, wl, steps, False, 0, 1)
        return sim, [wl.ops(OP_DTYPE, t, 1, c0, TYPES, flags) for t in range(steps)]

    streamed = Digest()
    sim, host_ops = make()
    fmt = _lib.JFMT_4
    dec = JournalDecoder(log2_window=30)
    for st in range(steps):
        sim.schedule(host_ops[st])
        sim.run_streamed((st + 1) * step_ns, lambda info, r, ev: streamed.add(ev), fmt=fmt,
                         buf_events=args.stream_events, decode=True, decoder=dec)
    st_s, now_s, round_s = sim.stats(), sim.now, sim.round
    sim.close()

    drained = Digest()
    sim, host_ops = make()
    cap = 1 << 24
    buf = np.zeros(cap, dtype=EVENT_DTYPE)

    def drain_all():
        while True:
            n = sim.drain_into(buf.ctypes.data, cap)
            drained.add(buf[:n])
            if n < cap:
                break
    for st in range(steps):
        sim.schedule(host_ops[st])
        while sim.run_raw((st + 1) * step_ns) == 1:
            drain_all()
        drain_all()
    assert drained.n == streamed.n == sim.journal_written() > 2 * 700_000_000
    assert streamed.sum == drained.sum
    assert sim.stats() == st_s and sim.now == now_s and sim.round == round_s
    sim.close()
