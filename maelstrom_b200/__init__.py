"""maelstrom_b200 -- H100-native replacement for Maelstrom's hot path
(maelstrom.process + maelstrom.net), behind the C ABI in
include/maelstrom_b200.h.  The Python layer here is only the host-side mirror
of the reference's interface for that path; all simulation work is CUDA."""
from . import _lib  # noqa: F401
from .engine import Sim, SimError, Config, TYPES, TOPOLOGIES, DISTS, body, kv_history, nemesis_grudge  # noqa: F401

__all__ = ["Sim", "SimError", "Config", "TYPES", "TOPOLOGIES", "DISTS", "body", "kv_history", "nemesis_grudge"]
