"""Placement at exclusive levels >= 1 on the H100 (DESIGN.md §3.9, RBGTOPO_CFG_LEVEL_PLACEMENT): every group of a fleet
that mixes levels 0..3 against the oracle's wave loop on the group's level view (levels_view), bit for bit — assign,
status, domain, and the dense rows and top-K keys of step batches — on every entry point that places at a level, plus
the error paths of the flag and of the level words."""
import os
import subprocess
import sys

import numpy as np
import pytest

import groups_gen as gg
import levels_oracle as lo
import levels_view as lvw
from alternates_oracle import run_fleet_ranked
from oracle import placer as oracle_placer
from oracle import wave_loop
from rbg_b200 import _lib, synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, BlobBuilder, Group, GroupsBuilder, Step
from rbg_b200.engine import RbgTopoError, TopoPlacer

pytestmark = pytest.mark.gpu

EINVAL, ELIMIT = -1, -6


def partitions(topo, seed, kind):
    """Levels 1..3: 'mixed' = hostname-like (one node per domain), one domain, a random nested level; 'edge' = domains of
    exactly 256 and 257 members, hostname-like; 'random' = levels_oracle.random_levels (nested and not)."""
    n = topo.n
    rng = np.random.default_rng(seed)
    if kind == "random":
        lv = lo.random_levels(rng, n, topo.domain, 3, [True, False, True])
    elif kind == "edge":
        d = np.zeros(n, np.int64)
        d[:min(n, 256)] = 0
        d[256:513] = 1
        d[513:] = 2 + np.arange(max(0, n - 513)) // 300
        perm = rng.permutation(n)
        l1 = np.empty(n, np.int64)
        l1[perm] = d
        _, l1 = np.unique(l1, return_inverse=True)
        lv = np.stack([topo.domain, l1, np.arange(n), np.zeros(n, np.int64)]).astype(np.int32)
    else:
        nested = lo.random_levels(rng, n, topo.domain, 1, [True])[1]
        lv = np.stack([topo.domain, np.arange(n), np.zeros(n, np.int64), nested]).astype(np.int32)
    nd = [len(topo.domain_owner)] + [int(lv[L].max()) + 1 for L in range(1, lv.shape[0])]
    return lv, nd


def fleet(seed, n, kind, scarce=False, fixed_level=True):
    """A groups_gen fleet with every group at a level in 0..3 (fixed domains renumbered into the group's level)."""
    case = gg.make_case(seed, n, scarce=scarce, exclusive=True)
    topo = case.topo
    lv, nd = partitions(topo, seed, kind)
    rng = np.random.default_rng(seed + 77)
    ng = int(case.blob[2])
    levels = [g % 4 for g in range(ng)]
    gb = lvw.with_levels(case.blob, levels)
    for g in range(ng):
        off = 8 + 12 * g + 2
        if gb[off] >= 0 and levels[g] > 0:  # a fixed domain of the group's own level
            gb[off] = int(rng.integers(0, nd[levels[g]])) if fixed_level else -1
    gids = [int(gb[8 + 12 * g]) for g in range(ng)]
    occ = lo.random_occ(np.random.default_rng(seed + 5), n, 3, gids[:4] + [999], max(1, n // 6))
    return topo, lv, nd, gb, occ


def engine(topo, **kw):
    eng = TopoPlacer(device=0, level_placement=True, **kw)
    eng.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    return eng


def offsets(gb):
    ng = int(gb[2])
    return np.concatenate([[0], np.cumsum([int(gb[8 + 12 * g + 9]) for g in range(ng)])]).astype(int)


def assert_fleet(res, exp, gb, where, staged=False):
    a, s, d = res
    offs = offsets(gb)
    for g in range(int(gb[2])):
        if staged and exp[g][1] == 1:  # the staged plan leaves non-gang groups with an unplaced replica at status 1
            assert int(s[g]) == 1, (where, g)
            continue
        assert (a[offs[g]:offs[g + 1]].tolist(), int(s[g]), int(d[g])) == exp[g], (where, g)


def staged(eng, gb):
    h = eng.stage_groups(gb)
    try:
        eng.run_staged(h, 1)
        return eng.fetch(h)
    finally:
        eng.release(h)


def bits(x):
    return np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)


def check_ranked(eng, gb, views, n_alt):
    """place_groups_ranked against tests/alternates_oracle.py on every group's level view: assign, status, domain, the
    replicas' scores, alternate nodes and their scores (the view's reported domain is 2 * domain)."""
    got = eng.place_groups_ranked(gb, n_alt)
    for x, y in zip(got[:3], eng.place_groups(gb)):
        assert np.array_equal(x, y)
    offs = offsets(gb)
    for g in range(int(gb[2])):
        exp = run_fleet_ranked(views[g], wave_loop.groups_from_blob(lo.groups_blob_for_view(gb, g)), n_alt)
        a, b = offs[g], offs[g + 1]
        ed = exp[2][g] // 2 if exp[2][g] >= 0 else -1
        assert np.array_equal(got[0][a:b], exp[0][a:b]) and int(got[1][g]) == int(exp[1][g]) and int(got[2][g]) == ed, g
        assert np.array_equal(bits(got[3][a:b]), bits(exp[3][a:b])), ("score", g)
        assert np.array_equal(got[4][a:b], exp[4][a:b]) and np.array_equal(bits(got[5][a:b]), bits(exp[5][a:b])), ("alt", g)


CASES = [(41, 1, "mixed"), (42, 33, "mixed"), (43, 33, "random"), (44, 2049, "mixed"), (45, 2049, "random"),
         (46, 4097, "edge"), (47, 4097, "random")]


@pytest.mark.parametrize("seed,n,kind", CASES)
def test_fleets_mixing_levels_match_the_oracle(seed, n, kind):
    """place_groups (direct) and stage_groups / run_staged, scarce and ample capacity, nested and non-nested levels."""
    topo, lv, nd, gb, occ = fleet(seed, n, kind, scarce=seed % 2 == 0)
    eng = engine(topo, chunk_nodes=128)
    try:
        eng.set_exclusive_levels(lv[1:], occ, level_n_domains=nd[1:])
        owner = lo.derive_level_owner(lv, occ)
        assert np.array_equal(eng.read_snapshot("level_owner"), owner)
        exp, views = lvw.expected_fleet(topo, lv, owner, nd, gb)
        assert_fleet(eng.place_groups(gb), exp, gb, "direct")
        assert_fleet(staged(eng, gb), exp, gb, "staged", staged=True)
        # ranked: the same placement, and every replica's score and alternates against alternates_oracle on the view
        check_ranked(eng, gb, views, 4)
        # an occupancy-only refresh and a capacity update between calls
        occ2 = lo.random_occ(np.random.default_rng(seed + 9), n, 3, [int(gb[8]), 998], max(1, n // 9))
        eng.set_exclusive_levels(None, occ2)
        free2 = np.maximum(topo.free - (np.arange(n) % 3 == 0), 0).astype(np.int32)
        eng.update_nodes(free=free2)
        topo2 = synth.Topology(topo.row_ptr, topo.col_idx, topo.edge_w, free2, topo.domain, topo.domain_owner)
        exp2, _ = lvw.expected_fleet(topo2, lv, lo.derive_level_owner(lv, occ2), nd, gb)
        assert_fleet(eng.place_groups(gb), exp2, gb, "direct after refresh")
    finally:
        eng.close()


def step_batch(topo, lv, nd, gids, seed):
    rng = np.random.default_rng(seed)
    steps = []
    for k, g in enumerate(gids):
        L = k % 4
        fixed = -1 if k % 3 else int(lv[L, int(rng.integers(0, topo.n))])
        steps.append(Step(gid=g, roles=[(3, 1, 2, ROLE_EXCLUSIVE), (2, 1, 1, 0)], pair=[[1, 1], [0, 1]],
                          anchors=[(int(rng.integers(0, topo.n)), 0, 1)], flags=STEP_EXCLUSIVE, fixed_domain=fixed,
                          level=L))
    # a hub-anchored step: the closed neighbourhoods of the hub and its neighbours make a large patched set
    hub = int(np.argmax(np.diff(topo.row_ptr)))
    steps.append(Step(gid=gids[0], roles=[(2, 1, 1, ROLE_EXCLUSIVE)], pair=[[1]],
                      anchors=[(int(c), 0, 1) for c in topo.col_idx[topo.row_ptr[hub]:topo.row_ptr[hub + 1]]][:200]
                      + [(hub, 0, 1)], flags=STEP_EXCLUSIVE, level=1))
    return steps


@pytest.mark.parametrize("n", [33, 2049])
def test_step_batches_match_the_oracle(n):
    """rbgtopo_score_assign and stage / run_staged: dense rows, top-K keys, assign, status and domain of every step
    against the oracle on its group's level view."""
    topo, lv, nd, gb, occ = fleet(60 + n, n, "random")
    gids = [int(gb[8 + 12 * g]) for g in range(int(gb[2]))]
    steps = step_batch(topo, lv, nd, gids, n)
    eng = engine(topo)
    try:
        eng.set_exclusive_levels(lv[1:], occ, level_n_domains=nd[1:])
        owner = lo.derive_level_owner(lv, occ)
        other = max(gids) + 1
        for st in steps:
            blob = BlobBuilder().add(st).build()
            view = lvw.level_view(topo, lv, owner, nd, st.level, st.gid, other)
            vst = Step(**{**st.__dict__, "fixed_domain": 2 * st.fixed_domain if st.fixed_domain >= 0 else -1,
                          "level": 0})
            ref = oracle_placer.place(view, BlobBuilder().add(vst).build(), want_matrix=True, want_topk=True)
            assert ref["rc"] == 0
            rd = [x // 2 if x >= 0 else -1 for x in ref["domain"]]
            a, s, d = eng.score_assign(blob)
            assert np.array_equal(a, ref["assign"]) and np.array_equal(s, ref["status"]) and list(d) == rd, st.level
            h = eng.stage(blob)
            try:
                eng.run_staged(h, 1)
                a, s, d = eng.fetch(h)
                assert np.array_equal(a, ref["assign"]) and list(d) == rd
                for row in range(ref["matrix"].shape[0]):
                    assert np.array_equal(eng.read_scores(h, row).view(np.uint32), ref["matrix"][row].view(np.uint32))
                for rr in range(len(st.roles)):
                    assert np.array_equal(eng.read_topk(h, rr), ref["topk"][rr]), rr
            finally:
                eng.release(h)
    finally:
        eng.close()


@pytest.mark.parametrize("world", [2, 4])
def test_replicated_ranks_match_the_oracle(world):
    """world > 1 contexts on one device: replicated selection gives every rank the oracle's placement."""
    topo, lv, nd, gb, occ = fleet(70 + world, 2049, "mixed")
    owner = lo.derive_level_owner(lv, occ)
    exp, _ = lvw.expected_fleet(topo, lv, owner, nd, gb)
    engs = [engine(topo, rank=r, world=world, chunk_nodes=128) for r in range(world)]
    try:
        for e in engs:
            e.set_exclusive_levels(lv[1:], occ, level_n_domains=nd[1:])
        for r, e in enumerate(engs):
            assert_fleet(e.place_groups(gb), exp, gb, f"rank {r}")
    finally:
        for e in engs:
            e.close()


def test_flagged_level0_fleets_equal_unflagged():
    """Level-0 fleets give byte-equal results with and without the flag (direct, staged, step batches)."""
    case = gg.make_case(81, 2049, exclusive=True)
    topo = case.topo
    lv, nd = partitions(topo, 81, "random")
    gids = [int(case.blob[8 + 12 * g]) for g in range(int(case.blob[2]))]
    occ = lo.random_occ(np.random.default_rng(81), topo.n, 3, gids[:4], 300)
    from gpu_util import new_engine
    e0, e1 = new_engine(topo), engine(topo)
    try:
        for e in (e0, e1):
            e.set_exclusive_levels(lv[1:], occ, level_n_domains=nd[1:])
        for f in ("place_groups", "place_groups_committed"):
            for x, y in zip(getattr(e0, f)(case.blob), getattr(e1, f)(case.blob)):
                assert np.array_equal(np.asarray(x), np.asarray(y)), f
        for x, y in zip(staged(e0, case.blob), staged(e1, case.blob)):
            assert np.array_equal(x, y)
        blob = BlobBuilder().add(Step(gid=gids[1], roles=[(3, 1, 2, ROLE_EXCLUSIVE)], pair=[[1]],
                                      flags=STEP_EXCLUSIVE)).build()
        for x, y in zip(e0.score_assign(blob), e1.score_assign(blob)):
            assert np.array_equal(x, y)
    finally:
        e0.close()
        e1.close()


def _rc(fn, *a):
    try:
        fn(*a)
        return 0
    except RbgTopoError as e:
        return e.code


def test_limits_and_errors_leave_the_ctx_usable():
    import ctypes as C
    lib = _lib.load()
    h = C.c_void_p()
    assert lib.rbgtopo_create(C.byref(_lib.Config(device=0, rank=0, world=1, flags=2)), C.byref(h)) == EINVAL
    topo = synth.make_topology(64, seed=9, tiers=2, owned_frac=0.0, max_free=4)
    lv, nd = partitions(topo, 9, "mixed")
    ok = GroupsBuilder().add(Group(gid=3, roles=[(0, 2, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE)).build()

    def grp(level, fixed=-1):
        return GroupsBuilder().add(Group(gid=3, roles=[(0, 2, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE,
                                         fixed_domain=fixed, level=level)).build()

    def step(level, fixed=-1):
        return BlobBuilder().add(Step(gid=3, roles=[(1, 1, 0, ROLE_EXCLUSIVE)], flags=STEP_EXCLUSIVE, level=level,
                                      fixed_domain=fixed)).build()

    eng = engine(topo)
    try:
        def ok_after():
            a, s, d = eng.place_groups(ok)
            assert int(s[0]) == 0
        assert _rc(eng.place_groups, grp(1)) == EINVAL                          # no levels installed
        ok_after()
        eng.set_exclusive_levels(lv[1:], [(0, 3, 2)], level_n_domains=nd[1:])
        for f in (eng.place_groups, eng.stage_groups):
            assert _rc(f, grp(4)) == EINVAL, f                                  # above n_levels
            assert _rc(f, grp(1, fixed=nd[1])) == EINVAL, f                     # fixed domain >= the level's count
            assert _rc(f, grp(2, fixed=1)) == EINVAL, f                         # level 2 has one domain
            ok_after()
        assert _rc(eng.place_groups_committed, grp(1)) == ELIMIT                # committed batches: level 0 only
        ok_after()
        assert _rc(eng.score_assign, step(4)) == EINVAL
        assert _rc(eng.score_assign, step(1, fixed=nd[1])) == EINVAL
        ok_after()
        a, s, d = eng.place_groups(grp(1, fixed=nd[1] - 1))                     # the last domain of level 1: fine
        assert int(s[0]) in (0, 1) and int(d[0]) in (-1, nd[1] - 1)
        a, s, d = eng.place_groups(grp(2))                                      # one domain: everything in it
        assert int(d[0]) == 0
    finally:
        eng.close()


@pytest.mark.parametrize("env", ["RBGTOPO_PER_WAVE_PLAN", "RBGTOPO_EMIT_TMA", "RBGTOPO_NO_DIRECT", "RBGTOPO_EMIT_STEPS",
                                 "RBGTOPO_VERIFY_PLAN"])
def test_other_paths_in_a_subprocess(env):
    """The per-wave fallback, the TMA and the step-major dense-matrix kernels, the staged path of place_groups and the
    plan self-check (device-expanded plan, emit and row tables == the host-built plan, level bits included) read their
    switches once when the library loads: the fleet and step tests again in a process with the switch set."""
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "gpu",
                        os.path.join(here, "test_gpu_levels_place.py::test_fleets_mixing_levels_match_the_oracle"),
                        os.path.join(here, "test_gpu_levels_place.py::test_step_batches_match_the_oracle")],
                       env={**os.environ, env: "1"}, capture_output=True, text=True, cwd=os.path.dirname(here))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]


def _gather(ptrs):
    """All-gather of one device buffer per rank on a single GPU (test_gpu_shard_single.py): concatenate, rank-major."""
    from test_gpu_shard_single import _gather as gather
    return gather(ptrs)


@pytest.mark.parametrize("world", [2, 4])
def test_all_gather_scheme_matches_the_oracle(world):
    """world = 2 / 4 contexts on one device, the all-gather scheme with a device-copy exchange (k_shard_select, k_merge's
    D*, k_greedy): step batches at levels 0..3 per step, and group plans wave by wave, against the oracle on the level
    views; every rank's slab of the dense rows too."""
    topo, lv, nd, gb, occ = fleet(90 + world, 2049, "mixed")
    owner = lo.derive_level_owner(lv, occ)
    gids = [int(gb[8 + 12 * g]) for g in range(int(gb[2]))]
    steps = step_batch(topo, lv, nd, gids, world)[:-1]
    other = max(gids) + 1
    refs = []
    for st in steps:
        view = lvw.level_view(topo, lv, owner, nd, st.level, st.gid, other)
        vst = Step(**{**st.__dict__, "fixed_domain": 2 * st.fixed_domain if st.fixed_domain >= 0 else -1, "level": 0})
        refs.append(oracle_placer.place(view, BlobBuilder().add(vst).build(), want_matrix=True))
    bb = BlobBuilder()
    for st in steps:
        bb.add(st)
    blob = bb.build()
    exp_fleet, _ = lvw.expected_fleet(topo, lv, owner, nd, gb)
    engs = [engine(topo, rank=r, world=world) for r in range(world)]
    try:
        for e in engs:
            e.set_exclusive_levels(lv[1:], occ, level_n_domains=nd[1:])
        # step batch
        hs = [e.stage(blob) for e in engs]
        allk = _gather([e.shard_score(h) for e, h in zip(engs, hs)])
        m = [e.shard_merge(h, allk.data_ptr()) for e, h in zip(engs, hs)]
        all2 = _gather([(x[1], x[2]) for x in m]) if m[0][0] else None
        for e, h in zip(engs, hs):
            e.shard_assign(h, all2.data_ptr() if all2 is not None else None)
        for r, (e, h) in enumerate(zip(engs, hs)):
            a, s, d = e.fetch(h)
            off, row = 0, 0
            lo_, hi = e.slab()
            for i, (st, ref) in enumerate(zip(steps, refs)):
                R = st.n_replicas
                rd = ref["domain"][0] // 2 if ref["domain"][0] >= 0 else -1
                assert a[off:off + R].tolist() == ref["assign"].tolist() and int(s[i]) == int(ref["status"][0]), (r, i)
                assert int(d[i]) == rd, (r, i)
                for k in range(R):
                    got = e.read_scores(h, row + k)
                    assert np.array_equal(got.view(np.uint32), ref["matrix"][k, lo_:hi].view(np.uint32)), (r, i, k)
                off += R
                row += R
            e.release(h)
        # group plans, wave by wave
        hs = [e.stage_groups(gb) for e in engs]
        for w in range(engs[0].shard_waves(hs[0])):
            allk = _gather([e.shard_wave_score(h, w) for e, h in zip(engs, hs)])
            m = [e.shard_wave_merge(h, w, allk.data_ptr()) for e, h in zip(engs, hs)]
            all2 = _gather([(x[1], x[2]) for x in m]) if m[0][0] else None
            for e, h in zip(engs, hs):
                e.shard_wave_assign(h, w, all2.data_ptr() if all2 is not None else None)
        for r, (e, h) in enumerate(zip(engs, hs)):
            assert_fleet(e.fetch(h), exp_fleet, gb, f"all-gather rank {r}", staged=True)
            e.release(h)
    finally:
        for e in engs:
            e.close()


def test_partition_install_makes_level_handles_stale():
    """A handle staged with groups at levels >= 1 belongs to the partitions it was validated against: after a new
    install it is refused (and can still be released); a level-0 handle keeps running."""
    topo, lv, nd, gb, occ = fleet(95, 2049, "mixed")
    gb0 = lvw.with_levels(gb, [0] * int(gb[2]))
    for g in range(int(gb[2])):
        if gb[8 + 12 * g + 2] >= nd[0]:
            gb0[8 + 12 * g + 2] = -1
    eng = engine(topo)
    try:
        eng.set_exclusive_levels(lv[1:], occ, level_n_domains=nd[1:])
        h1, h0 = eng.stage_groups(gb), eng.stage_groups(gb0)
        eng.set_exclusive_levels(lv[1:3], occ[occ[:, 2] <= 2], level_n_domains=nd[1:3])   # fewer levels
        assert _rc(eng.run_staged, h1, 1) != 0
        eng.release(h1)
        eng.run_staged(h0, 1)
        eng.fetch(h0)
        eng.release(h0)
        ok = GroupsBuilder().add(Group(gid=3, roles=[(0, 2, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE,
                                       level=1)).build()
        a, s, d = eng.place_groups(ok)                                                 # the new partitions place
        exp, _ = lvw.expected_fleet(topo, lv[:3], lo.derive_level_owner(lv[:3], occ[occ[:, 2] <= 2]), nd[:3], ok)
        assert (a.tolist(), int(s[0]), int(d[0])) == exp[0]
    finally:
        eng.close()
