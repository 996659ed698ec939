"""Multi-GPU host adapter: one process per GPU (torch.distributed), endpoints sharded by
index range (SURVEY.md section 8e).  The engine's kernels deliver cross-shard messages
by writing straight into the owner's inbox rings over NVLink peer memory (CUDA IPC,
include/maelstrom_b200.h "multi-GPU"); this module only supplies the plumbing the C ABI
asks for: the exchange of the IPC blobs and, optionally, a per-round NCCL barrier (a
1-element all-reduce enqueued on the engine's CUDA stream) instead of the engine's own
peer-memory barrier kernel."""
import ctypes as C

import numpy as np

from . import _lib
from .engine import Sim

EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)


def shard_owner(e, n_servers, n_shards):
    """Python restatement of owner_of() (csrc/ms_device.cuh); tests pin it to ms_shard_owner."""
    if n_shards <= 1:
        return 0
    if e < n_servers:
        return (e * n_shards) // n_servers
    return (e - n_servers) % n_shards


def merge_journals(parts):
    """parts: per-shard event arrays of equal length where foreign slots are 0xFF bytes.
    Returns the merged array; every slot must be produced by exactly one shard."""
    out = parts[0].copy()
    filled = parts[0]["event_id"] != EMPTY
    for p in parts[1:]:
        m = p["event_id"] != EMPTY
        if np.any(filled & m):
            raise ValueError("journal slot produced by two shards")
        out[m] = p[m]
        filled |= m
    if not np.all(filled):
        raise ValueError("journal slot produced by no shard")
    return out


def exchange_blobs(local_blob, group=None):
    """all_gather of the MS_SHARD_BLOB_BYTES blobs (works with gloo and nccl)."""
    import torch.distributed as dist
    blobs = [None] * dist.get_world_size(group)
    dist.all_gather_object(blobs, bytes(local_blob), group=group)
    return blobs


class ShardedSim:
    """engine.Sim for this rank's shard + the torch.distributed plumbing."""

    def __init__(self, n_nodes, group=None, device=None, nccl_barrier=False, **kw):
        import torch
        import torch.distributed as dist
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        if device is None:
            device = torch.cuda.current_device()
        self.device = device
        self.sim = Sim(n_nodes, n_shards=self.world, shard_id=self.rank, device=device, **kw)
        L, h = self.sim.L, self.sim.h
        blob = (C.c_ubyte * _lib.SHARD_BLOB_BYTES)()
        self.sim._chk(L.ms_shard_handles(h, blob))
        for peer, b in enumerate(exchange_blobs(blob, group)):
            buf = (C.c_ubyte * _lib.SHARD_BLOB_BYTES).from_buffer_copy(b)
            self.sim._chk(L.ms_shard_connect(h, peer, buf))
        self._flag = torch.zeros(1, device=torch.device("cuda", device))
        self._stream = torch.cuda.ExternalStream(int(L.ms_stream(h)), device=torch.device("cuda", device))

        def _barrier(ctx, stream_ptr):
            with torch.cuda.stream(self._stream):
                dist.all_reduce(self._flag, group=group)

        self._cb = _lib.BARRIER_FN(_barrier)          # keep a reference: C holds the pointer
        if nccl_barrier:
            self.sim._chk(L.ms_set_barrier(h, self._cb, None))
        # default: the engine's own k_barrier over NVLink peer flags (no host round trip per round)
        dist.barrier(group)

    def __getattr__(self, name):                      # add_endpoint, schedule, run, step, ...
        return getattr(self.sim, name)

    def set_origin(self, *args, **kw):
        """ms_set_origin on this rank's shard; every rank calls it with the same arguments (each shard sets its
        own endpoints' ring counters)."""
        return self.sim.set_origin(*args, **kw)

    def stats(self):
        """net.checker stats summed over the shards (every shard counts its own endpoints' events)."""
        import torch
        import torch.distributed as dist
        st = self.sim.stats()
        keys = [(c, k) for c in ("all", "clients", "servers") for k in ("send-count", "recv-count", "msg-count")]
        t = torch.tensor([st[c][k] for c, k in keys], dtype=torch.int64, device=self._flag.device)
        dist.all_reduce(t, group=self.group)
        out = {}
        for (c, k), v in zip(keys, t.tolist()):
            out.setdefault(c, {})[k] = int(v)
        return out

    def gather_journal(self):
        """Drain this shard's events and merge all shards' (every rank gets the full journal)."""
        import torch.distributed as dist
        ev, _ = self.sim.drain(bodies=False)
        parts = [None] * self.world
        dist.all_gather_object(parts, ev, group=self.group)
        return merge_journals(parts)

    def close(self):
        self.sim.close()
