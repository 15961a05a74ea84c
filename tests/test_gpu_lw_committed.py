"""GPU: committed leader-worker batches (rbgtopo_place_groups_lw_committed, DESIGN.md §3.13) bit for bit against the
oracle (tests/lw_committed_oracle.py) — assign per pod, status, domain — on seeded fleets with scarce capacity,
exclusive and gang groups, mixed S and C, co-location at levels 1 and 2, map and occupancy modes, shared gids, a fixed
domain another gid holds, a chain of many rounds and a refresh between calls; the reductions to
place_groups_committed and place_groups_lw; the rounds; every error code followed by a call that still works."""
import threading

import numpy as np
import pytest

import commit_gen as cg
import lw_commit_gen as lg
import lw_oracle as lw
from lw_committed_oracle import run_lw_committed
from rbg_b200 import synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, Group
from rbg_b200.engine import RbgTopoError, TopoPlacer

pytestmark = pytest.mark.gpu


def engine(topo, **kw):
    eng = TopoPlacer(device=0, **kw)
    eng.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    return eng


def fleet_engine(f: lg.Fleet, levels: bool):
    eng = engine(f.topo)
    if levels:
        eng.set_exclusive_levels(f.lv[1:], f.occ)
    return eng


def check(eng, topo, gblob, rp, **kw):
    a, s, d, rounds = eng.place_groups_lw_committed(gblob, rp)
    ea, es, ed = run_lw_committed(topo, gblob, rp, **kw)
    assert np.array_equal(a, ea), np.nonzero(a != ea)[0][:8]
    assert np.array_equal(s, es) and np.array_equal(d, ed), (s, es, d, ed)
    ng = int(gblob[2])
    assert (1 if ng else 0) <= rounds <= max(ng, 1), (rounds, ng)
    return a, s, d, rounds


@pytest.mark.parametrize("seed,n,scarce", lg.SEEDS)
@pytest.mark.parametrize("mode", ["map", "occupancy"])
def test_seeded_fleets(seed, n, scarce, mode):
    occ = mode == "occupancy"
    f = lg.fleet(seed, n, n_groups=14, scarce=scarce, levels=occ, occupancy=occ)
    eng = fleet_engine(f, occ)
    try:
        kw = dict(level_domain=list(f.lv), owner0=lg.owner0(f)) if occ else {}
        check(eng, f.topo, f.blob(), f.role_pods(), **kw)
    finally:
        eng.close()


def test_shared_gids_and_a_fixed_domain_another_gid_holds():
    """gid 7 reports domain d, gid 8 then fixes d, a later gid-7 group and a gid-8 group race for it: in map mode the
    claim hands d over to gid 8, in occupancy mode d is blocked for both (DESIGN.md §3.9's exception)."""
    topo = synth.make_topology(64, seed=5, tiers=2, max_free=4)
    topo.domain_owner[:] = -1
    d = int(topo.domain[0])
    mk = lambda gid, fixed=-1: Group(gid=gid, roles=[(0, 2, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE,
                                     fixed_domain=fixed)
    groups = [mk(7, d), mk(8, d), mk(7), mk(8), mk(7, d)]
    gb = lg.build(groups)
    rp = [(2, 0)] * len(groups)
    for occ in (False, True):
        eng = engine(topo)
        try:
            if occ:
                lv = np.stack([topo.domain, np.arange(64)]).astype(np.int32)
                eng.set_exclusive_levels(lv[1:], np.zeros((0, 3), np.int32))
                check(eng, topo, gb, rp, level_domain=list(lv), owner0=np.full(64, -1, np.int32))
            else:
                check(eng, topo, gb, rp)
        finally:
            eng.close()


def test_a_chain_runs_many_rounds():
    """Every group wants the same best node and takes what the one before it left: round after round the claims move."""
    case = cg.chain(24, 48, 3)
    rp = lw.role_pods_for(case.blob, lambda g, r: (2, -1))
    eng = engine(case.topo)
    try:
        _, _, _, rounds = check(eng, case.topo, case.blob, rp)
        assert rounds > 2
    finally:
        eng.close()


def test_refresh_between_calls():
    f = lg.fleet(21, 257, n_groups=10, scarce=True)
    eng = engine(f.topo)
    try:
        check(eng, f.topo, f.blob(), f.role_pods())
        rng = np.random.default_rng(0)
        f.topo.free = rng.integers(0, 4, f.topo.n).astype(np.int32)
        eng.update_nodes(f.topo.free)
        check(eng, f.topo, f.blob(), f.role_pods())
        nodes = np.arange(0, f.topo.n, 7, dtype=np.int32)
        f.topo.free[nodes] = 6
        eng.update_nodes_delta(nodes, f.topo.free[nodes])
        check(eng, f.topo, f.blob(), f.role_pods())
    finally:
        eng.close()


@pytest.mark.parametrize("k", range(len(cg.cases())))
def test_one_pod_per_replica_is_place_groups_committed(k):
    case = cg.cases()[k]
    eng = engine(case.topo)
    try:
        a, s, d, _ = eng.place_groups_lw_committed(case.blob, lw.role_pods_for(case.blob, lambda g, r: (1, -1)))
        ea, es, ed, _ = eng.place_groups_committed(case.blob)
        assert np.array_equal(a, ea) and np.array_equal(s, es) and np.array_equal(d, ed), case.name
    finally:
        eng.close()


def test_one_pod_per_replica_in_occupancy_mode():
    for case, lv, occ, _ in cg.occupancy_cases():
        eng = engine(case.topo)
        try:
            eng.set_exclusive_levels(lv[1:], occ)
            a, s, d, _ = eng.place_groups_lw_committed(case.blob, lw.role_pods_for(case.blob, lambda g, r: (1, -1)))
            ea, es, ed, _ = eng.place_groups_committed(case.blob)
            assert np.array_equal(a, ea) and np.array_equal(s, es) and np.array_equal(d, ed), case.name
        finally:
            eng.close()


def test_one_pod_per_replica_on_the_bench_fleet():
    import bench
    from rbg_b200.plugin import B200TopoPodGroupManager
    topo = synth.make_topology(4096, seed=3)
    eng = engine(topo)
    try:
        gblob, _ = B200TopoPodGroupManager(eng).groups_blob(bench.to_plugin(bench.fleet_spec("mooncake", 64, 4096, 3)))
        a, s, d, _ = eng.place_groups_lw_committed(gblob, lw.role_pods_for(gblob, lambda g, r: (1, -1)))
        ea, es, ed, _ = eng.place_groups_committed(gblob)
        assert np.array_equal(a, ea) and np.array_equal(s, es) and np.array_equal(d, ed)
    finally:
        eng.close()


@pytest.mark.parametrize("seed,n,scarce", lg.SEEDS[:4])
def test_group_zero_and_one_group_batches_are_place_groups_lw(seed, n, scarce):
    f = lg.fleet(seed, n, scarce=scarce)
    eng = engine(f.topo)
    try:
        a, s, d, _ = eng.place_groups_lw_committed(f.blob(), f.role_pods())
        ea, es, ed = eng.place_groups_lw(f.blob(), f.role_pods())
        n0 = sum(r[1] * sc[0] for r, sc in zip(f.groups[0].roles, f.rp[0]))
        assert np.array_equal(a[:n0], ea[:n0]) and s[0] == es[0] and d[0] == ed[0]
        for k in range(len(f.groups)):
            one = lg.Fleet(f.topo, [f.groups[k]], [f.rp[k]], f.lv, f.occ)
            a, s, d, rounds = eng.place_groups_lw_committed(one.blob(), one.role_pods())
            ea, es, ed = eng.place_groups_lw(one.blob(), one.role_pods())
            assert np.array_equal(a, ea) and np.array_equal(s, es) and np.array_equal(d, ed) and rounds == 1
    finally:
        eng.close()


def test_groups_that_cannot_meet_take_at_most_two_rounds():
    """Distinct fixed exclusive domains, each with room for its group."""
    topo = synth.make_topology(256, seed=9, tiers=2, max_free=8)
    topo.domain_owner[:] = -1
    doms = sorted(set(topo.domain.tolist()))[:6]
    groups = [Group(gid=20 + i, roles=[(0, 1, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE, fixed_domain=d)
              for i, d in enumerate(doms)]
    gb = lg.build(groups)
    eng = engine(topo)
    try:
        _, s, _, rounds = check(eng, topo, gb, [(2, 0)] * len(groups))
        assert (s == 0).all() and rounds <= 2
    finally:
        eng.close()


def _rc(fn, *a):
    try:
        fn(*a)
    except RbgTopoError as e:
        return e.code
    return 0


EINVAL, ELIMIT = -1, -6


def test_error_codes_leave_the_ctx_usable():
    f = lg.fleet(31, 64, n_groups=4)
    gb, rp = f.blob(), f.role_pods()
    lv = np.stack([f.topo.domain, np.arange(64) // 8]).astype(np.int32)
    lvl = Group(gid=3, roles=[(0, 1, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE, level=1)
    lvl_blob = lg.build(f.groups + [lvl])
    lvl_rp = np.concatenate([rp, [[2, -1]]])
    eng, flagged = engine(f.topo), engine(f.topo, committed_levels=True)
    try:
        assert _rc(eng.place_groups_lw_committed, gb, rp[:-1]) == EINVAL              # one role short
        bad = rp.copy()
        bad[0, 0] = 33
        assert _rc(eng.place_groups_lw_committed, gb, bad) == EINVAL                  # S above 32
        bad = rp.copy()
        bad[0, 1] = 1
        assert _rc(eng.place_groups_lw_committed, gb, bad) == EINVAL                  # level 1 not installed
        for e in (eng, flagged):
            e.set_exclusive_levels(lv[1:], np.zeros((0, 3), np.int32))
            assert _rc(e.place_groups_lw_committed, lvl_blob, lvl_rp) == ELIMIT        # exclusive at level 1
        check(eng, f.topo, gb, rp, level_domain=list(lv), owner0=np.full(64, -1, np.int32))
        check(flagged, f.topo, gb, rp, level_domain=list(lv), owner0=np.full(64, -1, np.int32))
    finally:
        eng.close()
        flagged.close()
    engs = [engine(f.topo, rank=r, world=2) for r in range(2)]
    try:
        for e in engs:
            assert _rc(e.place_groups_lw_committed, gb, rp) == ELIMIT
            e.place_groups(gb)
    finally:
        for e in engs:
            e.close()


def test_concurrent_callers_agree():
    f = lg.fleet(41, 513, n_groups=12, scarce=True)
    eng = engine(f.topo)
    try:
        ref = eng.place_groups_lw_committed(f.blob(), f.role_pods())
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
