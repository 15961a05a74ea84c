"""GPU: leader-worker placement (rbgtopo_place_groups_lw, DESIGN.md §3.11) bit for bit against the oracle
(tests/lw_oracle.py) — assign per pod, status, domain — on the generated fleets of tests/groups_gen.py, the mooncake
and fleet8 shapes with multi-pod prefill and decode, co-location at level 0, at a hostname-like level and at a rack
level, exclusive groups at another level with fixed domains, scarce capacity, replicas that fit nowhere, demand 0,
S = 32, mixed S, gang, N from 1 to 2049; the reduction to rbgtopo_place_groups on the bench fleet; every error code
followed by a call that still works."""
import numpy as np
import pytest

import groups_gen as gg
import lw_oracle as lw
from rbg_b200 import synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, STEP_GANG, Group, GroupsBuilder
from rbg_b200.engine import RbgTopoError, TopoPlacer

pytestmark = pytest.mark.gpu


def engine(topo, **kw):
    eng = TopoPlacer(device=0, **kw)
    eng.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    return eng


def build(groups):
    gb = GroupsBuilder()
    for g in groups:
        gb.add(g)
    return gb.build()


def check(eng, topo, gblob, rp, **kw):
    got = eng.place_groups_lw(gblob, rp)
    exp = lw.run_lw(topo, gblob, rp, **kw)
    assert np.array_equal(got[0], exp[0]), np.nonzero(got[0] != exp[0])[0][:8]
    assert np.array_equal(got[1], exp[1]) and np.array_equal(got[2], exp[2]), (got[1], exp[1], got[2], exp[2])
    return got


def cycle_pods(gblob, S=(2, 4, 1), C=(-1, 0)):
    k = iter(range(1 << 20))
    return lw.role_pods_for(gblob, lambda g, r: (S[(g + r) % len(S)], C[next(k) % len(C)]))


@pytest.mark.parametrize("seed,n,scarce,excl", gg.CASES)
def test_generated_fleets(seed, n, scarce, excl):
    case = gg.make_case(seed, n, scarce=scarce, exclusive=excl)
    eng = engine(case.topo)
    try:
        a, s, _ = check(eng, case.topo, case.blob, cycle_pods(case.blob))
        b, _, _ = check(eng, case.topo, case.blob, cycle_pods(case.blob, S=(4, 2), C=(0,)))
    finally:
        eng.close()


def test_one_node():
    topo = synth.make_topology(1, seed=1, tiers=1, max_free=8)
    topo.free[:] = 5
    g = Group(gid=3, roles=[(0, 2, 1, ROLE_EXCLUSIVE), (1, 2, 2, 0)], pair=[[1, 1], [1, 1]], flags=STEP_EXCLUSIVE)
    gblob = build([g, Group(gid=4, roles=[(0, 1, 0, 0)], pair=[[1]], flags=STEP_GANG)])
    eng = engine(topo)
    try:
        check(eng, topo, gblob, [(2, 0), (1, -1), (32, 0)])
    finally:
        eng.close()


@pytest.mark.parametrize("shape,seed", [("mooncake", 0), ("mooncake", 1), ("fleet8", 0), ("fleet8", 2)])
def test_fleet_shapes_with_multi_pod_prefill_and_decode(shape, seed):
    import bench
    from rbg_b200.plugin import B200TopoPodGroupManager
    topo = synth.make_topology(2049, seed=seed)
    eng = engine(topo)
    try:
        gblob, runs = B200TopoPodGroupManager(eng).groups_blob(bench.to_plugin(bench.fleet_spec(shape, 24, 2049, seed)))
        rp = []
        for i, g in enumerate(runs):
            for ri in g.order:
                name = g.rbg.roles[ri].name
                rp.append(((2, 4)[(i + seed) % 2] if "prefill" in name or "decode" in name else 1, (0, -1)[i % 3 == 2]))
        _, s, _ = check(eng, topo, gblob, rp)
        assert (s == 0).any()
    finally:
        eng.close()


def level_setup(n, seed):
    topo = synth.make_topology(n, seed=seed, tiers=2, max_free=4)
    topo.domain_owner[:] = -1
    lv = [topo.domain, np.arange(n, dtype=np.int32), (np.arange(n) // 16).astype(np.int32)]
    return topo, lv


def level_topo(topo, dom):
    return synth.Topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, dom.astype(np.int32),
                          np.full(int(dom.max()) + 1, -1, np.int32))


@pytest.mark.parametrize("seed,n", [(1, 33), (2, 130), (3, 2049)])
def test_colocation_and_exclusive_levels(seed, n):
    """Levels 1 (one domain per node) and 2 (racks of 16) installed without pods (occupancy mode, every owner free);
    exclusive groups at level 0 and at level 2, some with fixed domains, co-location at 0, 1 and 2."""
    topo, lv = level_setup(n, seed)
    rng = np.random.default_rng(seed)
    groups, levels = [], []
    for g in range(12):
        L = (0, 2, 0, 2)[g % 4] if g % 3 else 0
        nd = int(lv[L].max()) + 1
        excl = g % 3 != 1
        fixed = int(rng.integers(0, nd)) if excl and g % 5 == 0 else -1
        roles = [(0, int(rng.integers(1, 4)), int(rng.integers(0, 3)), ROLE_EXCLUSIVE),
                 (0, int(rng.integers(0, 3)), 1, ROLE_EXCLUSIVE if g % 2 else 0),
                 (1, int(rng.integers(1, 3)), 1, ROLE_EXCLUSIVE)]
        groups.append(Group(gid=10 + g, roles=roles, pair=[[1, 1, 0], [1, 1, 1], [0, 1, 1]],
                            anchors=[(int(rng.integers(0, n)), 0, 1)], flags=(STEP_EXCLUSIVE if excl else 0) |
                            (STEP_GANG if g % 4 == 3 else 0), fixed_domain=fixed, level=L))
        levels.append(L)
    gblob = build(groups)
    rp = lw.role_pods_for(gblob, lambda g, r: ((2, 3, 4)[(g + r) % 3], (0, 1, 2, -1)[(g + 2 * r) % 4]))
    eng = engine(topo, level_placement=True)
    try:
        eng.set_exclusive_levels(lv[1:], np.zeros((0, 3), np.int32))
        got = eng.place_groups_lw(gblob, rp)
        for L in (0, 2):
            mine = [g for g in range(len(groups)) if levels[g] == L]
            exp = lw.run_lw(level_topo(topo, lv[L]), gblob, rp, level_domain=lv, excl_domain=lv[L], groups=mine)
            sizes, k = [], 0
            for grp in groups:
                sizes.append(sum(r[1] * int(rp[k + i][0]) for i, r in enumerate(grp.roles)))
                k += len(grp.roles)
            offs = np.concatenate([[0], np.cumsum(sizes)])
            for g in mine:
                assert np.array_equal(got[0][offs[g]:offs[g + 1]], exp[0][offs[g]:offs[g + 1]]), (L, g)
                assert got[1][g] == exp[1][g] and got[2][g] == exp[2][g], (L, g, got[1][g], exp[1][g], got[2][g], exp[2][g])
        assert (got[2] >= 0).any() and (got[0] >= 0).any()
    finally:
        eng.close()


def test_scarce_capacity_takes_a_lower_domain():
    """The best-scoring domain has room for one pod; the replica of 3 pods goes to the next domain that holds it, and
    a replica of 9 pods fits nowhere next to ones that do."""
    n = 64
    topo = synth.make_topology(n, seed=4, tiers=2, max_free=1)
    topo.domain_owner[:] = -1
    topo.free[:] = 0
    topo.free[0:8] = [1, 0, 0, 0, 0, 0, 0, 0]
    topo.free[8:16] = 1
    g = Group(gid=1, roles=[(0, 2, 1, 0), (1, 1, 1, 0)], pair=[[1, 0], [0, 1]], anchors=[(0, 0, 4)])
    gblob = build([g, Group(gid=2, roles=[(0, 1, 1, 0)], pair=[[1]], anchors=[(0, 0, 4)])])
    eng = engine(topo)
    try:
        a, s, _ = check(eng, topo, gblob, [(3, 0), (9, 0), (4, 0)])
        assert ((a[:6] >= 8) & (a[:6] < 16)).all() and (a[6:15] < 0).all() and s.tolist() == [1, 0]
        assert ((a[15:] >= 8) & (a[15:] < 16)).all()
    finally:
        eng.close()


def test_demand_0_s32_mixed_sizes_anchors_and_gang():
    n = 130
    topo = synth.make_topology(n, seed=9, tiers=3, max_free=3)
    topo.domain_owner[:] = -1
    rng = np.random.default_rng(9)
    groups = [
        Group(gid=1, roles=[(0, 3, 0, 0)], pair=[[1]]),                                    # demand 0, S = 32
        Group(gid=2, roles=[(0, 2, 1, 0), (0, 3, 1, 0), (1, 2, 2, 0)], pair=[[1, 1, 1], [1, 1, 0], [1, 0, 2]],
              anchors=[(int(x), int(rng.integers(0, 3)), 2) for x in rng.choice(n, 5, replace=False)]),
        Group(gid=3, roles=[(0, 6, 2, 0)], pair=[[1]], flags=STEP_GANG),                   # gang that cannot fit
        Group(gid=4, roles=[(0, 2, 1, 0)], pair=[[1]], flags=STEP_GANG),                   # gang that fits
    ]
    gblob = build(groups)
    eng = engine(topo)
    try:
        for rp in ([(32, -1), (2, 0), (5, -1), (1, 0), (32, 0), (3, 0)],
                   [(32, 0), (1, -1), (4, 0), (3, -1), (16, -1), (2, -1)]):
            a, s, _ = check(eng, topo, gblob, rp)
        assert 2 in s.tolist() and 0 in s.tolist()
    finally:
        eng.close()


def test_one_pod_per_replica_is_place_groups_on_the_bench_fleet():
    import bench
    from rbg_b200.plugin import B200TopoPodGroupManager
    topo = synth.make_topology(10000, seed=0)
    eng = engine(topo)
    try:
        gblob, _ = B200TopoPodGroupManager(eng).groups_blob(bench.to_plugin(bench.fleet_spec("mooncake", 1024, 10000, 0)))
        rp = lw.role_pods_for(gblob, lambda g, r: (1, -1))
        got = eng.place_groups_lw(gblob, rp)
        exp = eng.place_groups(gblob)
        for x, y in zip(got, exp):
            assert np.array_equal(x, y)
    finally:
        eng.close()
    case = gg.make_case(5, 2049, scarce=True, exclusive=True)   # partial groups, gangs, exclusive domains
    eng = engine(case.topo)
    try:
        got = eng.place_groups_lw(case.blob, lw.role_pods_for(case.blob, lambda g, r: (1, -1)))
        for x, y in zip(got, eng.place_groups(case.blob)):
            assert np.array_equal(x, y)
    finally:
        eng.close()


def _code(fn):
    try:
        fn()
    except RbgTopoError as e:
        return e.code
    return 0


def test_error_codes_and_recovery():
    topo, lv = level_setup(130, 5)
    case = gg.make_case(2, 130, exclusive=True)
    gblob = case.blob
    rp = cycle_pods(gblob)
    eng = engine(case.topo)
    try:
        good = check(eng, case.topo, gblob, rp)

        def again():
            for x, y in zip(eng.place_groups_lw(gblob, rp), good):
                assert np.array_equal(x, y)

        for bad in ((0, -1), (33, -1), (2, -2), (2, 1)):   # S outside 1..32, C < -1, C above the (no) installed levels
            r2 = rp.copy()
            r2[1] = bad
            assert _code(lambda: eng.place_groups_lw(gblob, r2)) == -1, bad
            again()
        assert _code(lambda: eng.place_groups_lw(gblob, rp[:-1])) == -1    # role_pods of the wrong length
        again()
        rec, role_off = 8, int(gblob[8 + 4])
        for word, value in [(0, 0), (3, len(gblob) + 4), (2, -1), (rec + 1, 8), (rec + 3, 17), (rec + 8, 5),
                            (rec + 10, 1), (role_off + 1, -1), (role_off + 2, 1 << 20), (4, 1 << 20)]:
            b = gblob.copy()
            b[word] = value
            c1, c2 = _code(lambda: eng.place_groups(b)), _code(lambda: eng.place_groups_lw(b, rp))
            assert c1 == c2 and c1 != 0, (word, value, c1, c2)
            again()
    finally:
        eng.close()
    # C above the installed levels; a group at exclusive level >= 1 without RBGTOPO_CFG_LEVEL_PLACEMENT
    g = Group(gid=1, roles=[(0, 2, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE, level=2)
    g0 = Group(gid=2, roles=[(0, 2, 1, 0)], pair=[[1]])
    eng = engine(topo)
    try:
        eng.set_exclusive_levels(lv[1:], np.zeros((0, 3), np.int32))
        assert _code(lambda: eng.place_groups_lw(build([g0]), [(2, 3)])) == -1
        assert _code(lambda: eng.place_groups_lw(build([g]), [(2, 1)])) == -6
        check(eng, level_topo(topo, lv[0]), build([g0]), [(2, 2)], level_domain=lv)
    finally:
        eng.close()
    engs = [engine(case.topo, rank=r, world=2) for r in range(2)]
    try:
        for e in engs:
            assert _code(lambda: e.place_groups_lw(gblob, rp)) == -6
            e.place_groups(gblob)
    finally:
        for e in engs:
            e.close()
    fresh = TopoPlacer(device=0)
    try:
        assert _code(lambda: fresh.place_groups_lw(gblob, rp)) == -5
    finally:
        fresh.close()


def test_room_bitmap_beyond_48_kb_of_shared_memory():
    """400 000 nodes: the room bitmap takes 50 000 bytes of dynamic shared memory, more than a launch gets without
    the opt-in.  Domains of 50 000 nodes keep the oracle's enumeration of the co-location domains short."""
    n = 400_000
    topo = synth.make_topology(n, seed=2, tiers=2, max_free=2)
    topo.domain = (np.arange(n) // 50_000).astype(np.int32)
    topo.domain_owner = np.full(8, -1, np.int32)
    gblob = build([Group(gid=1, roles=[(0, 3, 1, 0), (1, 2, 1, 0)], pair=[[1, 1], [1, 1]], anchors=[(123456, 0, 1)]),
                   Group(gid=2, roles=[(0, 2, 2, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE | STEP_GANG)])
    eng = engine(topo)
    try:
        for rp in ([(4, -1), (2, -1), (3, -1)], [(4, 0), (2, 0), (8, 0)]):
            a, s, _ = check(eng, topo, gblob, rp)
            assert (a >= 0).all() and s.tolist() == [0, 0]
    finally:
        eng.close()


def test_exactness_bound_covers_waves_after_unplaced_pods():
    """A non-gang group of 40 one-pod replicas (two waves) whose wave 1 can see up to 16 unplaced pods of wave 0:
    each raises need by one (8 in the bound) and lowers the anchor weight by 1, so the bound is 152 + the scheduled
    pods' weight, not the 128 of a wave 0 that placed everything.  At the bound the call is refused before any wave
    runs; one below it, with capacity for 20 pods, it places and never meets an inexact wave."""
    n = 130
    topo = synth.make_topology(n, seed=6, tiers=2, max_free=1)
    topo.domain_owner[:] = -1
    topo.free[:] = 0
    topo.free[np.random.default_rng(6).choice(n, 20, replace=False)] = 1
    row_w = gg.wsum_max(topo) + 8000
    limit = ((1 << 24) + row_w - 1) // row_w

    def blob(c):
        return build([Group(gid=1, roles=[(0, 40, 1, 0)], pair=[[1]], anchors=[(7, 0, c)])])

    eng = engine(topo)
    try:
        for c in (limit - 152, limit - 140):
            assert _code(lambda: eng.place_groups_lw(blob(c), [(1, -1)])) == -4, c
        a, s, _ = check(eng, topo, blob(limit - 153), [(1, -1)])
        assert (a >= 0).sum() == 20 and s.tolist() == [1]
    finally:
        eng.close()
