"""Sharded engine on 2+ GPUs (one process per GPU, NCCL): the merged journal of all shards must
equal the oracle's (and therefore the single-GPU journal) bit for bit."""
import os
import socket

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, world, port, q, n, per_tick, latency_ms):
    import sys
    import traceback
    here = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, here)
    sys.path.insert(0, os.path.dirname(here))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        import oracle_lib as O
        from maelstrom_b200.engine import KIND_SIM_CLIENT
        from maelstrom_b200.sharded import ShardedSim
        from scenarios import random_broadcast_ops
        g = ShardedSim(n, workload="broadcast", topology="grid", n_values=4 * per_tick + 8, ring_cap=4096,
                       max_window=2048, journal_cap_log2=22, max_endpoints=n + 8,
                       latency_dist="constant", latency_mean_ms=latency_ms, journal_level=1)
        cs = [g.add_endpoint("c%d" % i, KIND_SIM_CLIENT) for i in range(3)]
        ops, nv = random_broadcast_ops(n, cs, n_ticks=3, per_tick=per_tick, seed=17)
        g.schedule(ops)
        g.run(40_000_000 if latency_ms else 4_000_000)
        ev = g.gather_journal()
        st = g.stats()
        rings = [None] * world
        dist.all_gather_object(rings, g.ring_counters())
        if rank == 0:
            o = O.Sim(n, workload=O.W_BROADCAST, topology="grid", n_values=4 * per_tick + 8,
                      latency_dist="constant", latency_mean_ms=latency_ms)
            for i in range(3):
                o.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT)
            o.schedule(ops)
            o.run(40_000_000 if latency_ms else 4_000_000)
            ev_o, _ = o.journal()
            assert len(ev) == len(ev_o), (len(ev), len(ev_o))
            for f in ("event_id", "time_ns", "msg_id", "src", "dest"):
                assert np.array_equal(ev[f], ev_o[f]), f
            assert st == o.stats()
            assert g.now == o.now and g.round == o.round
            # gossip across the row split claims compact ring space on the peer GPU: every shard reports its
            # own servers, together all server -> server broadcast sends (latency 0) or none (latency > 0)
            from scenarios import compact_total, oracle_gossip_sends
            got = sum(compact_total(rc) for rc in rings)
            ev_o, bd_o = o.journal()
            assert got == (oracle_gossip_sends(ev_o, bd_o, n) if latency_ms == 0 else 0), got
            if latency_ms == 0:
                assert got > 0
        q.put((rank, "ok"))
    except Exception:   # noqa: BLE001
        q.put((rank, "FAIL: " + traceback.format_exc()))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("n,per_tick,latency_ms", [(64, 200, 0), (100, 60, 2)])
def test_sharded_journal_equals_oracle(n, per_tick, latency_ms):
    import torch
    import torch.multiprocessing as mp
    world = min(torch.cuda.device_count(), 4)
    if world < 2:
        pytest.skip("needs at least 2 GPUs")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q, n, per_tick, latency_ms)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(r, "ok") for r in range(world)], res
