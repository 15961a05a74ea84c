"""GPU: ranked alternates of committed leader-worker batches at exclusive levels
(rbgtopo_place_groups_lw_committed_ranked on a ctx with RBGTOPO_CFG_LW_COMMIT_LEVELS, DESIGN.md §3.16): all seven
outputs bit for bit against tests/lw_committed_levels_oracle.py on seeded fleets, with co-location over the same
partitions; the one-pod and one-group reductions; a replay of two chunks at 2^20 nodes; NULL outputs."""
import numpy as np
import pytest

import lw_commit_levels_gen as lvg
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, Group
from rbg_b200.engine import TopoPlacer
from test_gpu_lw_committed_alternates import SENT, raw, same
from test_gpu_lw_limits import free_topo

pytestmark = pytest.mark.gpu


def engine(f: lvg.LvFleet, **kw):
    eng = TopoPlacer(device=0, **(kw or dict(lw_committed_levels=True)))
    t = f.topo
    eng.set_topology(t.row_ptr, t.col_idx, t.edge_w, t.free, t.domain, t.domain_owner)
    eng.set_exclusive_levels(f.lv[1:], f.occ)
    return eng


def check(eng, f: lvg.LvFleet, n_alts=(0, 3, 8), exp=None):
    gb, rp = f.blob(), f.role_pods()
    plain = eng.place_groups_lw_committed(gb, rp)
    exp = f.expected_ranked(8) if exp is None else exp
    same(plain[:3], exp[:3], "oracle placement")
    got = None
    for F in n_alts:
        got = eng.place_groups_lw_committed_ranked(gb, rp, F)
        same(got[:3], plain[:3], f"place_groups_lw_committed, n_alt {F}")
        assert got[3] == plain[3], (got[3], plain[3])
        same(got[4:], (exp[3], exp[4][:, :F], exp[5][:, :F]), f"oracle ranking, n_alt {F}")
    return got


@pytest.mark.parametrize("seed,n,scarce,kind", lvg.SEEDS)
def test_seeded_fleets(seed, n, scarce, kind):
    f = lvg.fleet(seed, n, n_groups=14, scarce=scarce, kind=kind)
    eng = engine(f)
    try:
        got = check(eng, f)
        assert (got[5] >= 0).any() or n < 16
    finally:
        eng.close()


@pytest.mark.parametrize("seed,n,scarce,kind", lvg.SEEDS[1:6])
def test_one_pod_per_replica_is_place_groups_committed_ranked(seed, n, scarce, kind):
    f = lvg.fleet(seed, n, n_groups=12, scarce=scarce, kind=kind)
    f.rp = [[(1, -1)] * len(rp) for rp in f.rp]
    eng, ref = engine(f), engine(f, committed_levels=True)
    try:
        got = eng.place_groups_lw_committed_ranked(f.blob(), f.role_pods(), 8)
        exp = ref.place_groups_committed_ranked(f.blob(), 8)
        same(got[:3] + got[4:], exp[:3] + exp[4:], "committed ranked")
    finally:
        eng.close()
        ref.close()


@pytest.mark.parametrize("seed,n,scarce,kind", lvg.SEEDS[2:6])
def test_one_group_batches_are_place_groups_lw_ranked(seed, n, scarce, kind):
    f = lvg.fleet(seed, n, n_groups=6, scarce=scarce, kind=kind)
    eng, ref = engine(f), engine(f, level_placement=True)
    try:
        for k in range(len(f.groups)):
            one = f.sub([k])
            got = eng.place_groups_lw_committed_ranked(one.blob(), one.role_pods(), 8)
            exp = ref.place_groups_lw_ranked(one.blob(), one.role_pods(), 8)
            same(got[:3] + got[4:], exp, f"group {k}")
            assert got[3] == 1
    finally:
        eng.close()
        ref.close()


def test_a_replay_of_two_chunks_at_two_to_the_twenty_nodes():
    """2^20 nodes, so a replay chunk holds 256 rows: 40 groups of one wave of 8 role rows make two chunks.  Odd groups
    are exclusive at level 0, zones of 64 nodes or hostnames in turn."""
    n = 1 << 20
    topo = free_topo(n, 17, max_free=2)
    topo.domain_owner[:] = -1
    topo.free[np.random.default_rng(17).random(n) > 0.01] = 0
    lv = np.stack([topo.domain, np.arange(n) // 64, np.arange(n)]).astype(np.int32)
    nd = [len(topo.domain_owner), n // 64, n]
    roles = [(0, 1, 1, ROLE_EXCLUSIVE)] * 8
    groups = [Group(gid=1 + g % 5, roles=roles, pair=[[1] * 8] * 8, anchors=[(int(g * 26_113 % n), 0, 1)],
                    flags=STEP_EXCLUSIVE if g % 2 else 0, level=(g // 2) % 3) for g in range(40)]
    rp = [[(2 if r == 0 else 1, -1) for r in range(8)] for _ in groups]
    f = lvg.LvFleet(topo, groups, rp, lv, nd, np.zeros((0, 3), np.int32))
    eng = engine(f)
    try:
        exp = f.expected_ranked(8)
        assert (exp[1] != 2).any()
        check(eng, f, n_alts=(8, 1), exp=exp)
        eng.place_groups_lw_committed(f.blob(), f.role_pods())
        plain = eng.last_timing()["launches"]
        eng.place_groups_lw_committed_ranked(f.blob(), f.role_pods(), 8)
        # the final lists (at most one k_set_heads) and two launches per chunk
        assert plain + 4 <= eng.last_timing()["launches"] <= plain + 5, (eng.last_timing()["launches"], plain)
    finally:
        eng.close()


def test_null_outputs():
    f = lvg.fleet(21, 257, n_groups=10, scarce=True, kind="random")
    gb, rp = f.blob(), f.role_pods()
    eng = engine(f)
    try:
        ref = check(eng, f, n_alts=(8,))
        P = len(ref[0])
        rc, out = raw(eng, gb, rp, 8, null_status=True)
        assert rc == 0 and (out["s"] == SENT).all()
        same((out["a"][:P], out["sc"][:P].view(np.float32), out["an"][:P * 8].reshape(P, 8),
              out["asc"][:P * 8].view(np.float32).reshape(P, 8)), (ref[0], ref[4], ref[5], ref[6]), "NULL status")
        rc, out = raw(eng, gb, rp, 0, null_status=True, null_alt=True)
        assert rc == 0
        same((out["a"][:P], out["sc"][:P].view(np.float32)), (ref[0], ref[4]), "n_alt 0, NULL alternates")
    finally:
        eng.close()
