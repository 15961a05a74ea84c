"""Occupancy mode on the H100 (DESIGN.md §3.9): the owner vectors k_level_owner derives, word for word against the numpy
derivation, level-0 placements against the existing oracle on each group's view of the snapshot, bit-identity with a ctx
given the equivalent domain-owner map, and the error paths of the level words."""
import numpy as np
import pytest

import groups_gen as gg
import levels_oracle as lo
from oracle import wave_loop
from rbg_b200 import synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, BlobBuilder, Group, GroupsBuilder, Step
from rbg_b200.engine import RbgTopoError

pytestmark = pytest.mark.gpu

EINVAL, ELIMIT = -1, -6


def levels_of(topo, seed, n_levels=3):
    rng = np.random.default_rng(seed)
    return lo.random_levels(rng, topo.n, topo.domain, n_levels, [True, False, True, False, True, False, True][:n_levels])


def occ_of(topo, seed, gids, n_levels, count=None):
    rng = np.random.default_rng(1000 + seed)
    return lo.random_occ(rng, topo.n, n_levels, gids, count if count is not None else max(1, topo.n // 8))


def test_derived_vectors_follow_every_refresh():
    from gpu_util import new_engine
    topo = synth.make_topology(700, seed=4, tiers=3, owned_frac=0.2, max_free=4)
    lv = levels_of(topo, 4, n_levels=7)
    eng = new_engine(topo)
    try:
        assert eng.read_snapshot("level_owner").size == 0
        occ = occ_of(topo, 4, [10, 11, 12], 7)
        eng.set_exclusive_levels(lv[1:], occ)
        assert np.array_equal(eng.read_snapshot("level_owner"), lo.derive_level_owner(lv, occ))
        occ2 = occ_of(topo, 5, [10, 13], 7, count=40)
        eng.set_exclusive_levels(None, occ2)                                   # occupancy only
        exp2 = lo.derive_level_owner(lv, occ2)
        assert np.array_equal(eng.read_snapshot("level_owner"), exp2)
        eng.update_nodes(free=np.maximum(topo.free - 1, 0))
        eng.update_nodes_delta([0, 5], [3, 0])
        assert np.array_equal(eng.read_snapshot("level_owner"), exp2)          # capacity does not move ownership
        eng.set_exclusive_levels(None, np.zeros((0, 3), np.int32))
        assert (eng.read_snapshot("level_owner") == -1).all()
        eng.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
        assert eng.read_snapshot("level_owner").size == 0                      # a new topology drops the levels
    finally:
        eng.close()


def _check_fleet(eng, topo, gblob, owner0, paths=("direct", "staged")):
    """Every group against the oracle's wave loop on its own view of the snapshot (levels_oracle.group_view)."""
    ng = int(gblob[2])
    gids = [int(gblob[8 + 12 * g]) for g in range(ng)]
    other = max(gids) + 1
    exp = []
    for g in range(ng):
        view = lo.group_view(topo, owner0, gids[g], other)
        states, _ = wave_loop.run_fleet(view, wave_loop.groups_from_blob(lo.groups_blob_for_view(gblob, g)))
        r = states[g].result()
        exp.append((states[g].assign_in_group_order(), r["status"], r["domain"] // 2 if r["domain"] >= 0 else -1))
    offs = np.concatenate([[0], np.cumsum([int(gblob[8 + 12 * g + 9]) for g in range(ng)])])
    if "direct" in paths:
        a, s, d = eng.place_groups(gblob)
        for g in range(ng):
            assert (a[offs[g]:offs[g + 1]].tolist(), int(s[g]), int(d[g])) == exp[g], ("direct", g)
    if "staged" in paths:
        h = eng.stage_groups(gblob)
        try:
            eng.run_staged(h, 1)
            a, s, d = eng.fetch(h)
        finally:
            eng.release(h)
        for g in range(ng):
            if exp[g][1] == 1:
                assert int(s[g]) == 1
                continue
            assert (a[offs[g]:offs[g + 1]].tolist(), int(s[g]), int(d[g])) == exp[g], ("staged", g)
    return exp


@pytest.mark.parametrize("seed,n", [(1, 1), (2, 7), (3, 33), (4, 130), (5, 2049)])
def test_level0_placements_match_the_oracle_in_occupancy_mode(seed, n):
    """Records at every level constrain level-0 groups (present / keyed terms), on the direct and staged paths."""
    from gpu_util import new_engine
    case = gg.make_case(seed, n, scarce=seed % 2 == 0, exclusive=True)
    topo = case.topo
    gids = [int(case.blob[8 + 12 * g]) for g in range(int(case.blob[2]))]
    lv = levels_of(topo, seed)
    occ = occ_of(topo, seed, gids[:4] + [999], 3, count=max(1, n // 6))
    eng = new_engine(topo)
    try:
        eng.set_exclusive_levels(lv[1:], occ)
        owner0 = lo.derive_level_owner(lv, occ)[0]
        assert np.array_equal(eng.read_snapshot("level_owner")[0], owner0)
        _check_fleet(eng, topo, case.blob, owner0)
    finally:
        eng.close()


def test_refresh_behind_an_in_flight_batch_sees_the_old_owners():
    from gpu_util import new_engine
    case = gg.make_case(11, 2049, exclusive=True)
    topo = case.topo
    lv = levels_of(topo, 11)
    gids = [int(case.blob[8 + 12 * g]) for g in range(int(case.blob[2]))]
    occ_a = occ_of(topo, 11, gids[:3], 3, count=300)
    occ_b = occ_of(topo, 12, gids[3:6], 3, count=300)
    eng = new_engine(topo)
    try:
        eng.set_exclusive_levels(lv[1:], occ_a)
        own_a = lo.derive_level_owner(lv, occ_a)[0]
        h = eng.stage_groups(case.blob)
        try:
            eng.run_staged(h, 3)                       # enqueued, not finished
            eng.set_exclusive_levels(None, occ_b)      # ordered behind them
            a, s, d = eng.fetch(h)
        finally:
            eng.release(h)
        ref = eng_results_for(topo, case.blob, own_a)
        ng = int(case.blob[2])
        offs = np.concatenate([[0], np.cumsum([int(case.blob[8 + 12 * g + 9]) for g in range(ng)])])
        for g in range(ng):
            if ref[g][1] != 1:
                assert (a[offs[g]:offs[g + 1]].tolist(), int(s[g]), int(d[g])) == ref[g], g
        assert np.array_equal(eng.read_snapshot("level_owner"), lo.derive_level_owner(lv, occ_b))
    finally:
        eng.close()


def eng_results_for(topo, gblob, owner0):
    ng = int(gblob[2])
    gids = [int(gblob[8 + 12 * g]) for g in range(ng)]
    out = []
    for g in range(ng):
        states, _ = wave_loop.run_fleet(lo.group_view(topo, owner0, gids[g], max(gids) + 1),
                                        wave_loop.groups_from_blob(lo.groups_blob_for_view(gblob, g)))
        r = states[g].result()
        out.append((states[g].assign_in_group_order(), r["status"], r["domain"] // 2 if r["domain"] >= 0 else -1))
    return out


@pytest.mark.parametrize("seed,n", [(21, 33), (22, 2049)])
def test_level0_records_equal_the_domain_owner_map(seed, n):
    """Level-0 records that imply a domain-owner map: bit-identical to a ctx given that map, on every entry point (the
    committed batch outside the corner of a fixed domain another gid holds)."""
    from gpu_util import new_engine
    case = gg.make_case(seed, n, exclusive=True)
    topo = case.topo
    rng = np.random.default_rng(seed)
    gids = [int(case.blob[8 + 12 * g]) for g in range(int(case.blob[2]))]
    nodes = rng.integers(0, n, max(1, n // 10))
    occ = np.array([(int(v), gids[int(topo.domain[v]) % len(gids)], 0) for v in nodes], dtype=np.int32).reshape(-1, 3)
    owner = lo.legacy_owner_map(topo.domain, len(topo.domain_owner), occ)
    legacy = synth.Topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, owner)
    e_old, e_new = new_engine(legacy), new_engine(topo)
    try:
        e_new.set_exclusive_levels([], occ)
        step = BlobBuilder().add(Step(gid=gids[1], roles=[(3, 1, 2, ROLE_EXCLUSIVE), (2, 1, 1, 0)], pair=[[1, 1], [0, 1]],
                                      flags=STEP_EXCLUSIVE)).build()
        # A committed batch differs in one corner (DESIGN.md §3.9): a group whose fixed domain another gid holds.  Its
        # claim blocks the domain for every later group in occupancy mode, and hands it over in the legacy map.
        outside = GroupsBuilder()
        for g in case.groups:
            if not (g.flags & STEP_EXCLUSIVE and g.fixed_domain >= 0 and owner[g.fixed_domain] not in (-1, g.gid)):
                outside.add(g)
        for f, gb in (("place_groups", case.blob), ("place_groups_committed", outside.build())):
            r_old, r_new = getattr(e_old, f)(gb), getattr(e_new, f)(gb)
            for x, y in zip(r_old, r_new):
                assert np.array_equal(np.asarray(x), np.asarray(y)), f
        for x, y in zip(e_old.score_assign(step), e_new.score_assign(step)):
            assert np.array_equal(x, y)
        h_old, h_new = e_old.stage_groups(case.blob), e_new.stage_groups(case.blob)
        e_old.run_staged(h_old), e_new.run_staged(h_new)
        for x, y in zip(e_old.fetch(h_old), e_new.fetch(h_new)):
            assert np.array_equal(x, y)
        for row in range(min(int(case.blob[4]), 40)):
            assert np.array_equal(e_old.read_scores(h_old, row).view(np.uint32), e_new.read_scores(h_new, row).view(np.uint32))
        e_old.release(h_old), e_new.release(h_new)
    finally:
        e_old.close()
        e_new.close()


def _rc(fn, *a):
    try:
        fn(*a)
        return 0
    except RbgTopoError as e:
        return e.code


def test_errors_leave_the_ctx_usable():
    from gpu_util import new_engine
    topo = synth.make_topology(64, seed=9, tiers=2, owned_frac=0.0, max_free=4)
    lv = levels_of(topo, 9, n_levels=2)
    ok = GroupsBuilder().add(Group(gid=3, roles=[(0, 2, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE)).build()

    def grp(level, fixed=-1):
        return GroupsBuilder().add(Group(gid=3, roles=[(0, 2, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE,
                                         fixed_domain=fixed, level=level)).build()

    def step(level):
        return BlobBuilder().add(Step(gid=3, roles=[(1, 1, 0, ROLE_EXCLUSIVE)], flags=STEP_EXCLUSIVE, level=level)).build()

    eng = new_engine(topo)
    try:
        def ok_after(code):
            assert code != 0
            a, s, d = eng.place_groups(ok)
            assert int(s[0]) == 0
        assert _rc(eng.place_groups, grp(1)) == EINVAL                          # no levels installed
        ok_after(-1)
        assert _rc(eng.score_assign, step(1)) == EINVAL
        assert _rc(eng.stage_groups, grp(1)) == EINVAL
        eng.set_exclusive_levels(lv[1:], [(0, 3, 2)])
        for f in (eng.place_groups, eng.place_groups_committed, eng.stage_groups):
            assert _rc(f, grp(1)) == ELIMIT, f                                  # installed: level-0 placement only
            assert _rc(f, grp(3)) == EINVAL, f                                  # above n_levels
            ok_after(-1)
        assert _rc(eng.score_assign, step(2)) == ELIMIT
        assert _rc(eng.score_assign, step(3)) == EINVAL
        assert _rc(eng.place_groups, grp(0, fixed=len(topo.domain_owner))) == EINVAL
        ok_after(-1)
        for bad in ([(64, 3, 0)], [(0, -1, 0)], [(0, 3, 3)], [(-1, 3, 0)]):
            assert _rc(eng.set_exclusive_levels, None, bad) == EINVAL, bad
            ok_after(-1)
        assert _rc(eng.set_exclusive_levels, lv[1:2], [(0, 3, 0)]) == 0         # a new partition set, one level
        assert _rc(eng.set_exclusive_levels, [np.full(64, 5, np.int32)], [], 0, [5]) == EINVAL   # domain >= count
        assert _rc(eng.update_nodes, None, topo.domain_owner) == EINVAL         # occupancy mode
        ok_after(-1)
        eng.update_nodes(free=topo.free)
        a, s, d = eng.place_groups(ok)
        assert int(s[0]) == 0
        assert np.array_equal(eng.read_snapshot("level_owner"), lo.derive_level_owner(lv[:2], [(0, 3, 0)]))
    finally:
        eng.close()


def test_step_batches_match_the_oracle_in_occupancy_mode():
    """rbgtopo_score_assign: every step against the oracle on its group's view of the snapshot."""
    from gpu_util import new_engine
    from oracle import placer as oracle_placer
    case = gg.make_case(31, 2049, exclusive=True)
    topo = case.topo
    gids = [int(case.blob[8 + 12 * g]) for g in range(int(case.blob[2]))]
    lv = levels_of(topo, 31)
    occ = occ_of(topo, 31, gids[:4], 3, count=400)
    rng = np.random.default_rng(31)
    steps = [Step(gid=g, roles=[(3, 1, 2, ROLE_EXCLUSIVE), (2, 1, 1, 0)], pair=[[1, 1], [0, 1]],
                  anchors=[(int(rng.integers(0, topo.n)), 0, 1)], flags=STEP_EXCLUSIVE,
                  fixed_domain=-1 if k % 3 else int(topo.domain[int(rng.integers(0, topo.n))])) for k, g in enumerate(gids)]
    eng = new_engine(topo)
    try:
        eng.set_exclusive_levels(lv[1:], occ)
        owner0 = lo.derive_level_owner(lv, occ)[0]
        bb = BlobBuilder()
        for st in steps:
            bb.add(st)
        a, s, d = eng.score_assign(bb.build())
        for k, st in enumerate(steps):
            view = lo.group_view(topo, owner0, st.gid, max(gids) + 1)
            one = Step(st.gid, st.roles, st.pair, st.anchors, st.consumed, st.flags,
                       2 * st.fixed_domain if st.fixed_domain >= 0 else -1)
            r = oracle_placer.place(view, BlobBuilder().add(one).build(), want_matrix=False, want_topk=False)
            assert r["rc"] == 0
            exp_d = int(r["domain"][0]) // 2 if r["domain"][0] >= 0 else -1
            assert (a[5 * k:5 * k + 5].tolist(), int(s[k]), int(d[k])) == (r["assign"].tolist(), int(r["status"][0]), exp_d), k
    finally:
        eng.close()


@pytest.mark.parametrize("world", [2, 4])
def test_replicated_ranks_match_the_oracle_in_occupancy_mode(world):
    """world > 1 contexts on one device: every rank holds the full-N owner vectors and returns the same placements."""
    from rbg_b200.engine import TopoPlacer
    case = gg.make_case(41, 2049, exclusive=True)
    topo = case.topo
    gids = [int(case.blob[8 + 12 * g]) for g in range(int(case.blob[2]))]
    lv = levels_of(topo, 41)
    occ = occ_of(topo, 41, gids[:4] + [999], 3, count=300)
    owner0 = lo.derive_level_owner(lv, occ)[0]
    engs = []
    try:
        for r in range(world):
            e = TopoPlacer(device=0, rank=r, world=world)
            engs.append(e)
            e.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
            e.set_exclusive_levels(lv[1:], occ)
            assert np.array_equal(e.read_snapshot("level_owner"), lo.derive_level_owner(lv, occ))
        for e in engs:
            _check_fleet(e, topo, case.blob, owner0)
    finally:
        for e in engs:
            e.close()


def test_per_wave_fallback_in_occupancy_mode():
    """The per-wave fallback (one launch per wave, no k_plan_group) on the same fleets, in a fresh process."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, RBGTOPO_PER_WAVE_PLAN="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "gpu",
                        os.path.join(root, "tests", "test_gpu_levels.py"), "-k", "level0_placements or fallback_plan_ctas"],
                       cwd=root, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert "6 passed" in r.stdout, r.stdout[-500:]


def test_fallback_plan_ctas():
    """Under RBGTOPO_PER_WAVE_PLAN the staged path runs without k_plan_group (plan_ctas == 0)."""
    import os
    from gpu_util import new_engine
    if not os.environ.get("RBGTOPO_PER_WAVE_PLAN"):
        pytest.skip("runs inside test_per_wave_fallback_in_occupancy_mode")
    case = gg.make_case(3, 33, exclusive=True)
    eng = new_engine(case.topo)
    try:
        eng.set_exclusive_levels([], [(0, int(case.blob[8]), 0)])
        h = eng.stage_groups(case.blob)
        eng.run_staged(h, 1)
        eng.fetch(h)
        eng.release(h)
        assert eng.stats()["plan_ctas"] == 0
    finally:
        eng.close()
