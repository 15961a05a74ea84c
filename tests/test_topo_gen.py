"""CPU: the irregular snapshots of tests/topo_gen.py are valid, reach every shape they are meant to reach, and the
plain numpy reference of the per-snapshot base vector agrees with the C oracle before any GPU test relies on it."""
import numpy as np
import pytest

import topo_gen as tg
from oracle import placer as oracle_placer
from rbg_b200.blob import BlobBuilder, Step


def test_seed_set_reaches_every_shape():
    seen = dict.fromkeys(tg.BULLETS, False)
    for name in tg.NAMES:
        for k, v in tg.coverage(tg.make(name)).items():
            seen[k] |= v
    missing = [k for k, v in seen.items() if not v]
    assert not missing, missing


@pytest.mark.parametrize("name", tg.NAMES)
def test_snapshot_is_valid(name):
    case = tg.make(name)
    t = case.topo
    assert oracle_placer.check_topology(t) == 0
    assert ((t.edge_w >= 0) & (t.edge_w <= tg.MAX_W)).all() and ((t.free >= 0) & (t.free <= tg.MAX_FREE)).all()
    if case.family in ("hubs", "sparse", "ties", "large") or name == "maxbase_bits":
        assert tg.wsum_max(t) <= 60000, tg.wsum_max(t)      # need up to 16 with a few anchors stays exact
    assert case.exact == (case.family != "inexact")


@pytest.mark.parametrize("name", [n for n in tg.NAMES if tg.BUILDERS[n][0] != "inexact"])
def test_base_ref_matches_the_oracle(name):
    """One role row, need 1, demand 0, no anchors: the oracle's dense row is W·min(free, 8) + 8000·min(free, 8)."""
    t = tg.make(name).topo
    blob = BlobBuilder().add(Step(gid=0, roles=[(1, 0, 1, 0)], pair=[])).build()
    ref = oracle_placer.place(t, blob, want_matrix=True, want_topk=False)
    assert ref["rc"] == 0
    exp = tg.base_ref(t)
    assert np.array_equal(ref["matrix"][0].view(np.uint32), exp.view(np.uint32))


def test_references_on_a_hand_example():
    """4 nodes: 0-1 (w 3), 1-2 (w 0), node 3 isolated; free 9, 2, 8, 0."""
    t = tg.from_edges(4, [0, 1], [1, 2], [3, 0], [9, 2, 8, 0])
    b = tg.base_ref(t)
    assert b.tolist() == [3 * 2 + 8000 * 8, 3 * 8 + 8000 * 2, 8000 * 8, 0]
    o = tg.order_ref(b)
    assert tg.key_node(o).tolist() == [0, 2, 1, 3]           # 64 006 and 64 000, then 16 024, then 0
    assert tg.pos_ref(o).tolist() == [0, 2, 1, 3]
    assert int(o[-1] >> np.uint64(32)) == 0x80000000 and int(o[-1] & np.uint64(0xFFFFFFFF)) == 0xFFFFFFFF - 3


def test_inexact_snapshot_sums_past_its_bound():
    """The bound of inexact_2p28 is 2^28 - 8 (28 bits); k_base's fp32 sum of the hub row is 2^28 (29 bits)."""
    t = tg.make("inexact_2p28").topo
    assert (tg.wsum_max(t) + tg.SELF_W) * tg.F_CAP == (1 << 28) - 8
    assert float(tg.k_base_fp32(t, 3)) == float(1 << 28)
