"""GPU: ranked placement (rbgtopo_place_groups_ranked, DESIGN.md §3.10) bit-equal to the oracle
(tests/alternates_oracle.py) run on the very same GROUPS blob — assign, status, domain, every replica's score and its
ranked alternates — and assign / status / domain equal to rbgtopo_place_groups on every input: contended batches,
the ABI limits of tests/groups_gen.py, exclusive fleets with fixed domains and opted-out roles, occupancy mode, groups
the host-driven loop re-runs, failed gangs, tables beyond shared memory and the bench fleet; n_alt 0, 1 and 8; the
staged and per-wave paths in subprocesses; every error path followed by a successful call."""
import os
import subprocess
import sys

import numpy as np
import pytest

import groups_gen as gg
import levels_oracle as lo
from alternates_oracle import run_fleet_ranked
from oracle import wave_loop
from rbg_b200 import synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_GANG, Group, GroupsBuilder
from rbg_b200.engine import RbgTopoError, TopoPlacer
from test_gpu_committed import contended_case

pytestmark = pytest.mark.gpu


def engine(topo, **kw):
    eng = TopoPlacer(device=0, **kw)
    eng.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    return eng


def bits(x):
    return np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)


def same(got, exp, R, ng):
    """got / exp: (assign, status, domain, score, alt_node, alt_score); the first R replicas and ng groups."""
    a, s, d, sc, an, asc = got
    ea, es, ed, esc, ean, easc = exp
    assert np.array_equal(a[:R], ea[:R]), np.nonzero(a[:R] != ea[:R])[0][:8]
    assert np.array_equal(s[:ng], es[:ng]) and np.array_equal(d[:ng], ed[:ng]), (s[:ng], es[:ng], d[:ng], ed[:ng])
    bad = np.nonzero(bits(sc[:R]) != bits(esc[:R]))[0]
    assert len(bad) == 0, ("score", bad[:8], sc[bad[:4]], esc[bad[:4]])
    bad = np.nonzero((an[:R] != ean[:R]).any(axis=1) | (bits(asc[:R]) != bits(easc[:R])).any(axis=1))[0]
    assert len(bad) == 0, ("alternates", bad[:8], an[bad[:2]], ean[bad[:2]], asc[bad[:2]], easc[bad[:2]])


def check(eng, topo, gblob, n_alt, limit=None):
    """The ranked call against place_groups and the oracle (the first `limit` groups: under snapshot semantics a
    group's result does not depend on the others)."""
    got = eng.place_groups_ranked(gblob, n_alt)
    plain = eng.place_groups(gblob)
    for x, y in zip(got[:3], plain):
        assert np.array_equal(x, y)
    assert got[4].shape == (len(got[0]), n_alt) and got[5].shape == (len(got[0]), n_alt)
    groups = wave_loop.groups_from_blob(gblob)[:limit]
    exp = run_fleet_ranked(topo, groups, n_alt)
    same(got, exp, len(exp[0]), len(groups))
    return got


def _build(groups):
    gb = GroupsBuilder()
    for g in groups:
        gb.add(g)
    return gb.build()


def test_contended_batches_match_oracle():
    """60 seeds of small contended batches (levels, gang and non-gang under scarce capacity, exclusive groups with
    preset and fixed domains, opted-out roles, shared gids, scheduled pods), n_alt cycling through 0, 1, 8."""
    seen = {"alts": 0, "partial": 0, "gang": 0, "excl": 0}
    for seed in range(60):
        topo, gblob = contended_case(seed, exclusive_all=seed % 3 == 0)
        eng = engine(topo)
        try:
            _, s, d, _, an, _ = check(eng, topo, gblob, (0, 1, 8)[seed % 3])
        finally:
            eng.close()
        seen["alts"] += int((an >= 0).sum())
        seen["partial"] += int((s == 1).sum())
        seen["gang"] += int((s == 2).sum())
        seen["excl"] += int((d >= 0).sum())
    assert all(seen.values()), seen


@pytest.mark.parametrize("seed,n,scarce,excl", gg.CASES)
def test_generated_fleets_at_the_abi_limits(seed, n, scarce, excl):
    case = gg.make_case(seed, n, scarce=scarce, exclusive=excl)
    eng = engine(case.topo)
    try:
        check(eng, case.topo, case.blob, 8)
    finally:
        eng.close()


def rerun_case(seed):
    """Non-gang groups whose first wave leaves replicas unplaced (more replicas than nodes with room), followed by a
    wave of a role with demand 0 that is always placed: the plan predicted that wave's `need` with every replica of
    the first wave placed, so place_groups re-runs these groups through the host-driven loop, and the rows that
    placed the second wave are that loop's, not the plan's."""
    rng = np.random.default_rng(seed)
    n = 64
    topo = synth.make_topology(n, seed=seed, tiers=2, max_free=1)
    room = rng.choice(n, size=5, replace=False)
    topo.free = np.zeros(n, np.int32)
    topo.free[room] = 1
    topo.domain_owner[:] = -1
    groups = []
    for i in range(8):
        a = 8 if i in (0, 5) else int(rng.integers(3, 9))
        flags = STEP_GANG if i == 5 else 0
        groups.append(Group(gid=10 + i, roles=[(0, a, 1, ROLE_EXCLUSIVE), (1, int(rng.integers(1, 4)), 0, ROLE_EXCLUSIVE)],
                            pair=[[1, 1], [1, 1]], anchors=[], flags=flags, fixed_domain=-1))
    return topo, _build(groups)


def test_groups_re_run_by_the_host_loop_rank_the_rows_that_placed_them():
    for seed in range(4):
        topo, gblob = rerun_case(seed)
        eng = engine(topo)
        try:
            _, s, _, sc, an, _ = check(eng, topo, gblob, 4)
            assert (s == 1).any() and (s == 2).any(), s       # re-run groups and a failed gang
            assert (an >= 0).any()
            # the plan's rows would be wrong here: `need` of the second wave differs from its prediction
            assert np.isfinite(sc).any()
        finally:
            eng.close()


def test_tables_beyond_shared_memory():
    """A group whose table of patched nodes does not fit k_plan_group's shared memory: place_groups takes the staged
    path with the per-wave selection kernels."""
    from test_gpu_groups_limits import _build as build_limits, _one_role_groups, _wide_group
    n = 4097
    rng = np.random.default_rng(120)
    topo = synth.make_topology(n, seed=3, tiers=4, max_free=4)
    wide = _wide_group(rng, 16, 5, n)
    p = np.asarray(wide.pair)
    p[:, 15] = 0
    wide.pair = p.tolist()
    wide.anchors = [(int(x), 15, 1) for x in rng.choice(n, size=120, replace=False)]
    groups = _one_role_groups(rng, 12, 10, n)
    groups.insert(3, wide)
    eng = engine(topo)
    try:
        check(eng, topo, build_limits(groups), 8)
    finally:
        eng.close()


@pytest.mark.parametrize("seed,n", [(3, 33), (4, 130)])
def test_occupancy_mode_fleets(seed, n):
    """Owners derived from exclusive pods at several levels: every group against the oracle on its own view of the
    snapshot (levels_oracle.group_view; the view's domains are 2 * domain + blocked, reported domains // 2)."""
    case = gg.make_case(seed, n, scarce=seed % 2 == 0, exclusive=True)
    topo, gblob = case.topo, case.blob
    ng = int(gblob[2])
    gids = [int(gblob[8 + 12 * g]) for g in range(ng)]
    lv = lo.random_levels(np.random.default_rng(seed), topo.n, topo.domain, 3, [True, False, True])
    occ = lo.random_occ(np.random.default_rng(1000 + seed), topo.n, 3, gids[:4] + [999], max(1, n // 6))
    eng = engine(topo)
    try:
        eng.set_exclusive_levels(lv[1:], occ)
        owner0 = lo.derive_level_owner(lv, occ)[0]
        got = eng.place_groups_ranked(gblob, 8)
        for x, y in zip(got[:3], eng.place_groups(gblob)):
            assert np.array_equal(x, y)
        offs = np.concatenate([[0], np.cumsum([int(gblob[8 + 12 * g + 9]) for g in range(ng)])])
        for g in range(ng):
            view = lo.group_view(topo, owner0, gids[g], max(gids) + 1)
            exp = run_fleet_ranked(view, wave_loop.groups_from_blob(lo.groups_blob_for_view(gblob, g)), 8)
            lo_, hi = offs[g], offs[g + 1]
            ed = exp[2][g] // 2 if exp[2][g] >= 0 else -1
            sl = lambda t: tuple(x[lo_:hi] for x in (t[0], t[3], t[4], t[5]))
            ga, gs_, gn, gas = sl(got)
            ea, es_, en, eas = sl(exp)
            assert np.array_equal(ga, ea) and int(got[1][g]) == int(exp[1][g]) and int(got[2][g]) == ed, g
            assert np.array_equal(bits(gs_), bits(es_)) and np.array_equal(gn, en) and np.array_equal(bits(gas), bits(eas)), g
    finally:
        eng.close()


def test_bench_fleet_mooncake_1024_groups_10000_nodes():
    """cfg3's fleet: the whole batch equal to place_groups, the first 160 groups against the oracle."""
    import bench
    from rbg_b200.plugin import B200TopoPodGroupManager
    topo = synth.make_topology(10000, seed=0)
    eng = engine(topo)
    try:
        gblob, _ = B200TopoPodGroupManager(eng).groups_blob(bench.to_plugin(bench.fleet_spec("mooncake", 1024, 10000, 0)))
        _, _, _, sc, an, _ = check(eng, topo, gblob, 8, limit=160)
        assert np.isfinite(sc).all() and (an >= 0).all()
    finally:
        eng.close()


def _code(fn):
    try:
        fn()
    except RbgTopoError as e:
        return e.code
    return 0


def test_error_paths_then_success_and_place_groups_unchanged_around_ranked_calls():
    topo, gblob = contended_case(11)
    eng = engine(topo)
    try:
        before = [x.copy() for x in eng.place_groups(gblob)]
        good = check(eng, topo, gblob, 2)
        for n_alt in (-1, 9):
            assert _code(lambda: eng.place_groups_ranked(gblob, n_alt)) == -1
            again = eng.place_groups_ranked(gblob, 2)
            assert all(np.array_equal(bits(x) if x.dtype == np.float32 else x, bits(y) if y.dtype == np.float32 else y)
                       for x, y in zip(again, good))
        rec = 8
        role_off = int(gblob[rec + 4])
        for word, value in [(0, 0), (1, 2), (3, len(gblob) + 4), (2, -1), (2, 100000), (rec + 1, 8), (rec + 2, 1 << 20),
                            (rec + 3, 0), (rec + 3, 17), (rec + 8, 5), (rec + 9, 1 << 20), (rec + 10, 1),
                            (role_off + 1, -1), (role_off + 2, 1 << 20), (role_off + 3, 4), (4, 1 << 20)]:
            b = gblob.copy()
            b[word] = value
            c1 = _code(lambda: eng.place_groups(b))
            c2 = _code(lambda: eng.place_groups_ranked(b, 8))
            assert c1 == c2 and c1 != 0, (word, value, c1, c2)
            again = eng.place_groups_ranked(gblob, 2)
            assert np.array_equal(again[4], good[4]) and np.array_equal(bits(again[3]), bits(good[3]))
        after = eng.place_groups(gblob)
        assert all(np.array_equal(x, y) for x, y in zip(before, after))
    finally:
        eng.close()
    fresh = TopoPlacer(device=0)
    try:
        assert _code(lambda: fresh.place_groups_ranked(gblob, 2)) == _code(lambda: fresh.place_groups(gblob)) == -5
    finally:
        fresh.close()
    engs = [engine(topo, rank=r, world=2) for r in range(2)]
    try:
        for e in engs:
            assert _code(lambda: e.place_groups_ranked(gblob, 2)) == -6
            assert all(np.array_equal(x, y) for x, y in zip(e.place_groups(gblob), before))
    finally:
        for e in engs:
            e.close()


@pytest.mark.parametrize("switch", ["RBGTOPO_NO_DIRECT", "RBGTOPO_PER_WAVE_PLAN"])
def test_staged_and_per_wave_paths(switch):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, **{switch: "1"})
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "gpu",
                        os.path.join(root, "tests", "test_gpu_alternates.py"),
                        "-k", "contended or abi_limits or re_run or beyond_shared or occupancy"],
                       cwd=root, env=env, capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert " passed" in r.stdout and "failed" not in r.stdout, r.stdout[-2000:]
