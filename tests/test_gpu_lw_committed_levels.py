"""GPU: committed leader-worker batches at exclusive levels (rbgtopo_place_groups_lw_committed on a ctx with
RBGTOPO_CFG_LW_COMMIT_LEVELS, DESIGN.md §3.16) bit for bit against tests/lw_committed_levels_oracle.py — assign per
pod, status, domain — on seeded fleets at N = 1 .. 4 097 over three partition kinds; the flag changing nothing at level
0; the one-pod and one-group reductions; a round that only a claim across levels causes; a chain of many rounds;
partition reinstalls and refreshes between calls; concurrent callers; every error code."""
import ctypes as C
import threading

import numpy as np
import pytest

import commit_gen as cg
import lw_commit_gen as lg
import lw_commit_levels_gen as lvg
from rbg_b200 import _lib, synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, Group
from rbg_b200.engine import RbgTopoError, TopoPlacer

pytestmark = pytest.mark.gpu

EINVAL, ELIMIT = -1, -6


def engine(topo, lv=None, occ=None, **kw):
    eng = TopoPlacer(device=0, **kw)
    eng.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    if lv is not None:
        eng.set_exclusive_levels(lv[1:], np.zeros((0, 3), np.int32) if occ is None else occ)
    return eng


def lv_engine(f: lvg.LvFleet):
    return engine(f.topo, f.lv, f.occ, lw_committed_levels=True)


def check(eng, f: lvg.LvFleet):
    gb, rp = f.blob(), f.role_pods()
    a, s, d, rounds = eng.place_groups_lw_committed(gb, rp)
    ea, es, ed = f.expected()
    assert np.array_equal(a, ea), np.nonzero(a != ea)[0][:8]
    assert np.array_equal(s, es) and np.array_equal(d, ed), (s, es, d, ed)
    ng = int(gb[2])
    assert (1 if ng else 0) <= rounds <= max(ng, 1), (rounds, ng)
    assert lvg.violations(f.lv, f.occ, gb, rp, a, s) == []
    return a, s, d, rounds


@pytest.mark.parametrize("seed,n,scarce,kind", lvg.SEEDS)
def test_seeded_fleets(seed, n, scarce, kind):
    f = lvg.fleet(seed, n, n_groups=14, scarce=scarce, kind=kind)
    eng = lv_engine(f)
    try:
        check(eng, f)
    finally:
        eng.close()


@pytest.mark.parametrize("seed,n,scarce", lg.SEEDS)
@pytest.mark.parametrize("mode", ["map", "occupancy"])
def test_the_flag_changes_nothing_at_level_zero(seed, n, scarce, mode):
    """lw_commit_gen's level-0 fleets: results, rounds and launches with the flag are those without it."""
    occ = mode == "occupancy"
    f = lg.fleet(seed, n, n_groups=14, scarce=scarce, levels=occ, occupancy=occ)
    out = []
    for kw in (dict(committed_levels=True), dict(lw_committed_levels=True)):
        eng = engine(f.topo, f.lv if occ else None, f.occ if occ else None, **kw)
        try:
            r = eng.place_groups_lw_committed(f.blob(), f.role_pods())
            out.append((r, eng.last_timing()["launches"]))
        finally:
            eng.close()
    (r0, l0), (r1, l1) = out
    assert all(np.array_equal(x, y) for x, y in zip(r0[:3], r1[:3])) and r0[3] == r1[3] and l0 == l1


@pytest.mark.parametrize("seed,n,scarce,kind", lvg.SEEDS[1:6])
def test_one_pod_per_replica_is_place_groups_committed(seed, n, scarce, kind):
    f = lvg.fleet(seed, n, n_groups=12, scarce=scarce, kind=kind)
    f.rp = [[(1, -1)] * len(rp) for rp in f.rp]
    eng, ref = lv_engine(f), engine(f.topo, f.lv, f.occ, committed_levels=True)
    try:
        a, s, d, _ = eng.place_groups_lw_committed(f.blob(), f.role_pods())
        ea, es, ed, _ = ref.place_groups_committed(f.blob())
        assert np.array_equal(a, ea) and np.array_equal(s, es) and np.array_equal(d, ed)
    finally:
        eng.close()
        ref.close()


@pytest.mark.parametrize("seed,n,scarce,kind", lvg.SEEDS[2:6])
def test_one_group_batches_are_place_groups_lw(seed, n, scarce, kind):
    f = lvg.fleet(seed, n, n_groups=8, scarce=scarce, kind=kind)
    eng, ref = lv_engine(f), engine(f.topo, f.lv, f.occ, level_placement=True)
    try:
        for k in range(len(f.groups)):
            one = f.sub([k])
            a, s, d, rounds = eng.place_groups_lw_committed(one.blob(), one.role_pods())
            ea, es, ed = ref.place_groups_lw(one.blob(), one.role_pods())
            assert np.array_equal(a, ea) and np.array_equal(s, es) and np.array_equal(d, ed) and rounds == 1
    finally:
        eng.close()
        ref.close()


def small(n=64):
    topo = synth.make_topology(n, seed=3, tiers=2, max_free=8)
    topo.domain_owner[:] = -1
    topo.free[:] = 4
    lv = np.stack([topo.domain, np.arange(n), np.arange(n) // 16]).astype(np.int32)
    return topo, lv, [len(topo.domain_owner), n, (n + 15) // 16]


def test_one_more_round_from_a_claim_across_levels():
    """A hostname-keyed group takes the best node; a zone-keyed group picks that node's zone in round 1, learns of the
    pod (P) in round 2 and moves, so the group after it runs a third round.  The same batch with the zone group not
    exclusive takes two."""
    topo, lv, nd = small()
    host = Group(gid=2, roles=[(0, 1, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE, level=1)
    zone = Group(gid=1, roles=[(0, 1, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE, level=2)
    tail = Group(gid=3, roles=[(0, 1, 1, 0)], pair=[[1]])
    f = lvg.LvFleet(topo, [host, zone, tail], [[(1, -1)], [(2, -1)], [(1, -1)]], lv, nd, np.zeros((0, 3), np.int32))
    eng = lv_engine(f)
    try:
        a, _, _, rounds = check(eng, f)
        assert lv[2][a[1]] != lv[2][a[0]] and rounds == 3, (a, rounds)
        g = f.groups[1]
        f.groups[1] = Group(gid=g.gid, roles=g.roles, pair=g.pair, flags=0, level=2)
        _, _, _, rounds = check(eng, f)
        assert rounds == 2
    finally:
        eng.close()


def test_a_chain_of_many_rounds():
    """commit_gen's chain with its groups at hostname, zone and level 0 in turn: round after round the claims move."""
    case = cg.chain(24, 48, 3)
    n = case.topo.n
    topo = case.topo
    topo.domain_owner[:] = -1
    lv = np.stack([topo.domain, np.arange(n), np.arange(n) // 4]).astype(np.int32)
    nd = [len(topo.domain_owner), n, (n + 3) // 4]
    groups = [Group(gid=grp.gid, roles=grp.roles, pair=grp.pair, anchors=grp.anchors, flags=STEP_EXCLUSIVE,
                    level=(1, 2, 0)[g % 3]) for g, grp in enumerate(case.groups)]
    f = lvg.LvFleet(topo, groups, [[(1, -1)] * len(g.roles) for g in groups], lv, nd, np.zeros((0, 3), np.int32))
    eng = lv_engine(f)
    try:
        _, _, _, rounds = check(eng, f)
        assert rounds > 2
    finally:
        eng.close()


def test_partitions_reinstalled_and_refreshes_between_calls():
    f = lvg.fleet(21, 257, n_groups=10, scarce=True, kind="mixed")
    eng = lv_engine(f)
    try:
        check(eng, f)
        g = lvg.fleet(21, 257, n_groups=10, scarce=True, kind="random")
        f.lv, f.nd, f.occ = g.lv, g.nd, g.occ
        eng.set_exclusive_levels(f.lv[1:], f.occ)
        f.groups = [Group(gid=x.gid, roles=x.roles, pair=x.pair, anchors=x.anchors, flags=x.flags,
                          fixed_domain=x.fixed_domain if x.level == 0 else -1, level=x.level) for x in f.groups]
        check(eng, f)
        rng = np.random.default_rng(0)
        f.topo.free = rng.integers(0, 4, f.topo.n).astype(np.int32)
        eng.update_nodes(f.topo.free)
        check(eng, f)
        nodes = np.arange(0, f.topo.n, 7, dtype=np.int32)
        f.topo.free[nodes] = 6
        eng.update_nodes_delta(nodes, f.topo.free[nodes])
        check(eng, f)
    finally:
        eng.close()


def test_concurrent_callers_agree():
    f = lvg.fleet(41, 513, n_groups=12, scarce=True, kind="edge")
    eng = lv_engine(f)
    try:
        ref = check(eng, f)
        out = [None] * 8

        def run(i):
            out[i] = eng.place_groups_lw_committed(f.blob(), f.role_pods())

        th = [threading.Thread(target=run, args=(i,)) for i in range(8)]
        for t in th:
            t.start()
        for t in th:
            t.join()
        for o in out:
            assert all(np.array_equal(x, y) for x, y in zip(o[:3], ref[:3])) and o[3] == ref[3]
    finally:
        eng.close()


def create_rc(flags):
    lib = _lib.load()
    cfg = _lib.Config(device=0, rank=0, world=1, slots=0, emit_matrix=1, chunk_nodes=0, flags=flags)
    h = C.c_void_p()
    rc = lib.rbgtopo_create(C.byref(cfg), C.byref(h))
    if rc == 0:
        lib.rbgtopo_destroy(h)
    return rc


def _rc(fn, *a):
    try:
        fn(*a)
    except RbgTopoError as e:
        return e.code
    return 0


def test_error_codes_leave_the_ctx_usable():
    assert [create_rc(fl) for fl in (4, 5, 6, 7, 3)] == [EINVAL, EINVAL, EINVAL, 0, 0]
    f = lvg.fleet(31, 64, n_groups=4, kind="mixed")
    gb, rp = f.blob(), f.role_pods()
    eng = lv_engine(f)
    try:
        bad = lvg.LvFleet(f.topo, f.groups + [Group(gid=3, roles=[(0, 1, 1, ROLE_EXCLUSIVE)], pair=[[1]],
                                                    flags=STEP_EXCLUSIVE, level=4)], f.rp + [[(1, -1)]], f.lv, f.nd, f.occ)
        assert _rc(eng.place_groups_lw_committed, bad.blob(), bad.role_pods()) == EINVAL   # L > n_levels
        check(eng, f)
    finally:
        eng.close()
    engs = [TopoPlacer(device=0, rank=r, world=2, lw_committed_levels=True) for r in range(2)]
    try:
        for e in engs:
            e.set_topology(f.topo.row_ptr, f.topo.col_idx, f.topo.edge_w, f.topo.free, f.topo.domain,
                           f.topo.domain_owner)
            e.set_exclusive_levels(f.lv[1:], f.occ)
        for e in engs:
            assert _rc(e.place_groups_lw_committed, gb, rp) == ELIMIT
    finally:
        for e in engs:
            e.close()


def test_one_node_past_the_room_bitmap():
    from test_gpu_lw_limits import BITMAP_NODES, free_topo
    m = BITMAP_NODES + 1
    topo = free_topo(m, 31, max_free=2)
    topo.domain_owner[:] = -1
    lv = np.stack([topo.domain, np.arange(m) // 16]).astype(np.int32)
    groups = [Group(gid=1, roles=[(0, 2, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE, level=1)]
    gb = lg.build(groups)
    eng = engine(topo, lv, lw_committed_levels=True)
    try:
        assert _rc(eng.place_groups_lw_committed, gb, [(2, -1)]) == ELIMIT
        assert _rc(eng.place_groups_lw_committed_ranked, gb, [(2, -1)], 8) == ELIMIT
        a, s, _, _ = eng.place_groups_committed(gb)
        assert s.tolist() == [0] and ((a >= 0) & (a < m)).all()
    finally:
        eng.close()
