"""GPU: ranked alternates for leader-worker pods (rbgtopo_place_groups_lw_ranked, DESIGN.md §3.12) bit for bit
(float bits) against the oracle (tests/lw_alternates_oracle.py) — assign, status, domain, every pod's score and its
ranked alternates — with assign / status / domain equal to rbgtopo_place_groups_lw's on every input: the generated
fleets of tests/groups_gen.py with mixed S and C, the mooncake and fleet8 shapes, co-location at level 0, at a
hostname level and at a rack level beside exclusive groups at another level with fixed domains, occupancy mode,
scarce capacity, demand 0, S = 32, gang failure, N = 1, 2049 and 400 000; the reduction to
rbgtopo_place_groups_ranked on the bench fleet; every error code followed by a call that works."""
import ctypes as C

import numpy as np
import pytest

import groups_gen as gg
import levels_oracle as lo
import lw_oracle as lw
from lw_alternates_oracle import groups_of, run_lw_ranked
from rbg_b200 import synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, STEP_GANG, Group
from rbg_b200.engine import RbgTopoError, TopoPlacer
from test_gpu_lw import build, cycle_pods, level_setup, level_topo
from test_oracle_lw_alternates import HAND_CASES

pytestmark = pytest.mark.gpu


def engine(topo, **kw):
    eng = TopoPlacer(device=0, **kw)
    eng.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    return eng


def bits(x):
    return np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)


def same(got, exp, pods=None, groups=None):
    """got / exp: the six outputs; pods / groups: index arrays to compare (default all)."""
    pods = np.arange(len(exp[0])) if pods is None else pods
    groups = np.arange(len(exp[1])) if groups is None else groups
    a, s, d, sc, an, asc = got
    ea, es, ed, esc, ean, easc = exp
    assert np.array_equal(a[pods], ea[pods]), pods[np.nonzero(a[pods] != ea[pods])[0][:8]]
    assert np.array_equal(s[groups], es[groups]) and np.array_equal(d[groups], ed[groups]), (s, es, d, ed)
    bad = pods[np.nonzero(bits(sc[pods]) != bits(esc[pods]))[0]]
    assert len(bad) == 0, ("score", bad[:8], sc[bad[:4]], esc[bad[:4]])
    bad = pods[np.nonzero((an[pods] != ean[pods]).any(axis=1) | (bits(asc[pods]) != bits(easc[pods])).any(axis=1))[0]]
    assert len(bad) == 0, ("alternates", bad[:8], an[bad[:2]], ean[bad[:2]], asc[bad[:2]], easc[bad[:2]])


def ranked(eng, gblob, rp, n_alt):
    """The ranked call, its assign / status / domain checked against place_groups_lw."""
    got = eng.place_groups_lw_ranked(gblob, rp, n_alt)
    for x, y in zip(got[:3], eng.place_groups_lw(gblob, rp)):
        assert np.array_equal(x, y)
    assert got[4].shape == (len(got[0]), n_alt) and got[5].shape == (len(got[0]), n_alt)
    return got


def check(eng, topo, gblob, rp, n_alt, **kw):
    got = ranked(eng, gblob, rp, n_alt)
    same(got, run_lw_ranked(topo, gblob, rp, n_alt, **kw))
    return got


def group_pods(gblob, rp, gs):
    G = groups_of(gblob, rp)
    return np.concatenate([np.arange(G[g].pod0, G[g].pod0 + G[g].n_pods) for g in gs] + [np.zeros(0, np.int64)])


@pytest.mark.parametrize("seed,n,scarce,excl", gg.CASES)
def test_generated_fleets(seed, n, scarce, excl):
    case = gg.make_case(seed, n, scarce=scarce, exclusive=excl)
    eng = engine(case.topo)
    seen = 0
    try:
        for k, F in enumerate((0, 1, 3, 8)):
            rp = cycle_pods(case.blob) if k % 2 == 0 else cycle_pods(case.blob, S=(4, 2), C=(0,))
            got = check(eng, case.topo, case.blob, rp, F)
            seen += int((got[4] >= 0).sum())
    finally:
        eng.close()
    assert seen > 0 or n == 1


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
        got = check(eng, topo, gblob, rp, (3, 8)[seed % 2])
        assert (got[4] >= 0).any() and (got[1] == 0).any()
    finally:
        eng.close()


@pytest.mark.parametrize("seed,n", [(1, 33), (2, 130), (3, 2049)])
def test_colocation_and_exclusive_levels(seed, n):
    """Levels 1 (one domain per node) and 2 (racks of 16); exclusive groups at levels 0 and 2, some with fixed
    domains, co-location at 0, 1 and 2 (test_gpu_lw's fleet), each group against the oracle at its own level."""
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
        for F in (2, 8):
            got = ranked(eng, gblob, rp, F)
            for L in (0, 2):
                mine = [g for g in range(len(groups)) if levels[g] == L]
                exp = run_lw_ranked(level_topo(topo, lv[L]), gblob, rp, F, level_domain=lv, excl_domain=lv[L],
                                    groups=mine)
                same(got, exp, group_pods(gblob, rp, mine), np.asarray(mine))
        assert (got[2] >= 0).any() and (got[4] >= 0).any()
    finally:
        eng.close()


@pytest.mark.parametrize("seed,n", [(3, 33), (4, 130)])
def test_occupancy_mode(seed, n):
    """Owners derived from exclusive pods at several levels: every group against the oracle on its own view of the
    snapshot (levels_oracle.group_view: domains 2 * domain + blocked, reported domains // 2); co-location reads the
    installed partitions themselves."""
    case = gg.make_case(seed, n, scarce=seed % 2 == 0, exclusive=True)
    topo, gblob = case.topo, case.blob
    ng = int(gblob[2])
    gids = [int(gblob[8 + 12 * g]) for g in range(ng)]
    lv = lo.random_levels(np.random.default_rng(seed), topo.n, topo.domain, 3, [True, False, True])
    occ = lo.random_occ(np.random.default_rng(1000 + seed), topo.n, 3, gids[:4] + [999], max(1, n // 6))
    rp = lw.role_pods_for(gblob, lambda g, r: ((2, 1, 3)[(g + r) % 3], (0, -1, 1, 3)[(g + r) % 4]))
    eng = engine(topo)
    try:
        eng.set_exclusive_levels(lv[1:], occ)
        owner0 = lo.derive_level_owner(lv, occ)[0]
        got = ranked(eng, gblob, rp, 8)
        for g in range(ng):
            view = lo.group_view(topo, owner0, gids[g], max(gids) + 1)
            exp = list(run_lw_ranked(view, lo.groups_blob_for_view(gblob, g), rp, 8, level_domain=lv, groups=[g]))
            exp[2] = np.where(exp[2] >= 0, exp[2] // 2, exp[2])
            same(got, exp, group_pods(gblob, rp, [g]), np.asarray([g]))
    finally:
        eng.close()


def test_scarce_capacity_demand_0_s32_and_gang():
    n = 130
    topo = synth.make_topology(n, seed=9, tiers=3, max_free=3)
    topo.domain_owner[:] = -1
    rng = np.random.default_rng(9)
    gblob = build([
        Group(gid=1, roles=[(0, 3, 0, 0)], pair=[[1]]),                                    # demand 0, S = 32
        Group(gid=2, roles=[(0, 2, 1, 0), (0, 3, 1, 0), (1, 2, 2, 0)], pair=[[1, 1, 1], [1, 1, 0], [1, 0, 2]],
              anchors=[(int(x), int(rng.integers(0, 3)), 2) for x in rng.choice(n, 5, replace=False)]),
        Group(gid=3, roles=[(0, 6, 2, 0)], pair=[[1]], flags=STEP_GANG),                   # gang that cannot fit
        Group(gid=4, roles=[(0, 2, 1, 0)], pair=[[1]], flags=STEP_GANG),                   # gang that fits
    ])
    eng = engine(topo)
    try:
        for rp, F in (([(32, -1), (2, 0), (5, -1), (1, 0), (32, 0), (3, 0)], 8),
                      ([(32, 0), (1, -1), (4, 0), (3, -1), (16, -1), (2, -1)], 3)):
            got = check(eng, topo, gblob, rp, F)
            assert 2 in got[1].tolist() and 0 in got[1].tolist()
    finally:
        eng.close()
    # scarce: the best domain holds one pod, a replica of 9 pods fits nowhere
    topo = synth.make_topology(64, seed=4, tiers=2, max_free=1)
    topo.domain_owner[:] = -1
    topo.free[:] = 0
    topo.free[0:16] = [1, 0, 0, 0, 0, 0, 0, 0] + [1] * 8
    gblob = build([Group(gid=1, roles=[(0, 2, 1, 0), (1, 1, 1, 0)], pair=[[1, 0], [0, 1]], anchors=[(0, 0, 4)]),
                   Group(gid=2, roles=[(0, 1, 1, 0)], pair=[[1]], anchors=[(0, 0, 4)])])
    eng = engine(topo)
    try:
        check(eng, topo, gblob, [(3, 0), (9, 0), (4, 0)], 8)
        check(eng, topo, gblob, [(2, -1), (1, -1), (3, -1)], 8)
    finally:
        eng.close()


def test_hand_built_known_answers():
    """The CPU file's known-answer cases (tests/test_oracle_lw_alternates.py) on the device."""
    for name, make in HAND_CASES.items():
        c = make()
        eng = engine(c["topo"], level_placement=True)
        try:
            if c.get("levels") is not None:
                eng.set_exclusive_levels(c["levels"], np.zeros((0, 3), np.int32))
            got = check(eng, c["topo"], c["blob"], c["rp"], c["n_alt"], level_domain=c.get("level_domain"))
            c["expect"](got)
        finally:
            eng.close()


def test_one_node_and_2049_nodes():
    topo = synth.make_topology(1, seed=1, tiers=1, max_free=8)
    topo.free[:] = 5
    g = Group(gid=3, roles=[(0, 2, 1, ROLE_EXCLUSIVE), (1, 2, 2, 0)], pair=[[1, 1], [1, 1]], flags=STEP_EXCLUSIVE)
    gblob = build([g, Group(gid=4, roles=[(0, 1, 0, 0)], pair=[[1]], flags=STEP_GANG)])
    eng = engine(topo)
    try:
        for F in (0, 8):
            check(eng, topo, gblob, [(2, 0), (1, -1), (32, 0)], F)
    finally:
        eng.close()
    case = gg.make_case(5, 2049, scarce=True, exclusive=True)
    eng = engine(case.topo)
    try:
        check(eng, case.topo, case.blob, cycle_pods(case.blob, S=(3, 1, 2), C=(0, -1, -1)), 8)
    finally:
        eng.close()


def test_room_bitmap_beyond_48_kb_of_shared_memory():
    n = 400_000
    topo = synth.make_topology(n, seed=2, tiers=2, max_free=2)
    topo.domain = (np.arange(n) // 50_000).astype(np.int32)
    topo.domain_owner = np.full(8, -1, np.int32)
    gblob = build([Group(gid=1, roles=[(0, 3, 1, 0), (1, 2, 1, 0)], pair=[[1, 1], [1, 1]], anchors=[(123456, 0, 1)]),
                   Group(gid=2, roles=[(0, 2, 2, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE | STEP_GANG)])
    eng = engine(topo)
    try:
        for rp in ([(4, -1), (2, -1), (3, -1)], [(4, 0), (2, 0), (8, 0)]):
            got = check(eng, topo, gblob, rp, 8)
            assert (got[0] >= 0).all() and (got[4] >= 0).all()
    finally:
        eng.close()


def test_one_pod_per_replica_is_place_groups_ranked_on_the_bench_fleet():
    import bench
    from rbg_b200.plugin import B200TopoPodGroupManager
    topo = synth.make_topology(10000, seed=0)
    eng = engine(topo)
    try:
        gblob, _ = B200TopoPodGroupManager(eng).groups_blob(bench.to_plugin(bench.fleet_spec("mooncake", 1024, 10000, 0)))
        rp = lw.role_pods_for(gblob, lambda g, r: (1, -1))
        for F in (0, 8):
            got = eng.place_groups_lw_ranked(gblob, rp, F)
            exp = eng.place_groups_ranked(gblob, F)
            for x, y in zip(got, exp):
                assert x.dtype == y.dtype and x.tobytes() == y.tobytes()
    finally:
        eng.close()


def _code(fn):
    try:
        fn()
    except RbgTopoError as e:
        return e.code
    return 0


def test_error_codes_and_recovery():
    case = gg.make_case(2, 130, exclusive=True)
    gblob = case.blob
    rp = cycle_pods(gblob)
    eng = engine(case.topo)
    try:
        good = check(eng, case.topo, gblob, rp, 3)

        def again():
            for x, y in zip(eng.place_groups_lw_ranked(gblob, rp, 3), good):
                assert x.tobytes() == y.tobytes()

        for F in (-1, 9):
            assert _code(lambda: eng.place_groups_lw_ranked(gblob, rp, F)) == -1, F
            again()
        for bad in ((0, -1), (33, -1), (2, -2), (2, 1)):
            r2 = rp.copy()
            r2[1] = bad
            assert _code(lambda: eng.place_groups_lw_ranked(gblob, r2, 3)) == -1, bad
            again()
        assert _code(lambda: eng.place_groups_lw_ranked(gblob, rp[:-1], 3)) == -1
        again()
        gb, r = np.ascontiguousarray(gblob, np.int32), np.ascontiguousarray(rp.reshape(-1), np.int32)
        out = np.empty(4096, np.int32)
        p = lambda a: a.ctypes.data_as(C.POINTER(C.c_int32))
        f32 = np.empty(4096, np.float32).ctypes.data_as(C.POINTER(C.c_float))
        lib = eng.lib
        assert lib.rbgtopo_place_groups_lw_ranked(eng._h, p(gb), len(gb), p(r), len(r), 3, p(out), None, None, None,
                                                  p(out), f32) == -1     # NULL score
        again()
        assert lib.rbgtopo_place_groups_lw_ranked(eng._h, p(gb), len(gb), p(r), len(r), 3, p(out), None, None, f32,
                                                  None, f32) == -1       # NULL alt_node with n_alt > 0
        again()
        assert lib.rbgtopo_place_groups_lw_ranked(eng._h, p(gb), len(gb), None, 0, 3, p(out), None, None, f32,
                                                  p(out), f32) == -1     # NULL role_pods
        again()
        # status / domain may be NULL; alt_* may be NULL with n_alt = 0
        sc = np.empty(len(good[0]), np.float32)
        a = np.empty(len(good[0]), np.int32)
        assert lib.rbgtopo_place_groups_lw_ranked(eng._h, p(gb), len(gb), p(r), len(r), 0, p(a), None, None,
                                                  sc.ctypes.data_as(C.POINTER(C.c_float)), None, None) == 0
        assert np.array_equal(a, good[0]) and bits(sc).tobytes() == bits(good[3]).tobytes()
    finally:
        eng.close()
    engs = [engine(case.topo, rank=k, world=2) for k in range(2)]
    try:
        for e in engs:
            assert _code(lambda: e.place_groups_lw_ranked(gblob, rp, 3)) == -6
            e.place_groups(gblob)
    finally:
        for e in engs:
            e.close()
    fresh = TopoPlacer(device=0)
    try:
        assert _code(lambda: fresh.place_groups_lw_ranked(gblob, rp, 3)) == -5
    finally:
        fresh.close()
