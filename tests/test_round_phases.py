"""k_round's emission phase (PE2, DESIGN.md 3.5) against the oracle at journal level 2.  In a window that
qualifies for per-neighbor ring claims, gossip emissions take the compact fast path and every other emission
(a reply) the general one, from the same loop; these cases put both kinds, in every mix, into the same windows:

- broadcasts with a msg_id (the broadcast_ok reply is the message's LAST emission), without one (gossip
  only) and reads (a reply only), injected round after round so that they share windows with the gossip of
  earlier rounds;
- grid (a value reaches a node from 2 to 4 neighbors in one round), line, and tree4 (degree 5: past the
  four register compares of the source slot);
- loss > 0 and latency > 0, where no window qualifies and the general path does all the work.

Every case runs on the emulator ([emul], CPU suite) and on the H100 ([cuda])."""
import numpy as np
import pytest

import oracle_lib as O
from scenarios import assert_same_journal, both, compact_total, make_pair, oracle_gossip_sends

pytestmark = pytest.mark.usefixtures("engine_backend")


def flood(n, topo, mix, rounds=4, per_round=40, seed=3, **net):
    g, o = make_pair(n, topology=topo, n_values=rounds * per_round + 8, ring_cap=4096, max_window=2048,
                     journal_cap_log2=20, journal_level=2, max_endpoints=n + 8, **net)

    def scenario(s, body):
        rng = np.random.default_rng(seed)
        cs = [s.add_endpoint("c%d" % i, O.KIND_SIM_CLIENT) for i in range(2)]
        mid = 0
        v = 0
        for _ in range(rounds):
            for _ in range(per_round):
                c = cs[int(rng.integers(2))]
                dest = int(rng.integers(n))
                kind = mix[int(rng.integers(len(mix)))]
                mid += 1
                if kind == "id":
                    s.send(c, dest, body("broadcast", msg_id=mid, p0=v))
                    v += 1
                elif kind == "plain":
                    s.send(c, dest, body("broadcast", p0=v))
                    v += 1
                else:
                    s.send(c, dest, body("read", msg_id=mid))
            s.step(1)
        s.run(400_000_000)

    both(g, o, scenario)
    return g, o


@pytest.mark.parametrize("topo,n", [("grid", 25), ("line", 9), ("tree4", 40)])
@pytest.mark.parametrize("mix", [("plain",), ("id",), ("id", "plain", "read")], ids=["plain", "id", "mixed"])
def test_gossip_and_replies_share_windows(topo, n, mix):
    g, o = flood(n, topo, mix)
    ev, bd = o.journal()
    want = oracle_gossip_sends(ev, bd, n)
    got = compact_total(g.ring_counters())
    assert want > 500
    if topo == "tree4":
        assert 0 < got <= want          # degree 5: compact only for block-ordered windows
    else:
        assert got == want              # every gossip record went into ring space claimed per neighbor
    assert_same_journal(g, o)
    for k in range(n):
        assert np.array_equal(g.node_set(k), o.node_set(k))


@pytest.mark.parametrize("net", [dict(p_loss=0.2), dict(latency_dist="constant", latency_mean_ms=2)],
                         ids=["loss", "latency"])
def test_non_qualifying_windows_take_the_general_path(net):
    g, o = flood(25, "grid", ("id", "plain", "read"), **net)
    assert compact_total(g.ring_counters()) == 0
    assert_same_journal(g, o)
