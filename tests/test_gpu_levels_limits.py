"""GPU: exclusive topology at the key a group names, at its limits (DESIGN.md §3.9), bit for bit against the oracles.

The cases come from tests/levels_limits_cases.py.  The derived owner vectors (read_snapshot("level_owner")) are
checked word for word against levels_oracle.derive_level_owner_fast after every install and refresh: k_level_owner
past its first grid stride in all three phases, the ⊕-merge under thousands of gids on one domain, partition
reinstalls that grow the tables, and the total domain ceiling.  Placement at keys 4..7 — the upper half of the 3-bit
level fields of the step flags, the row table and the group record — is checked on every entry point that places at
a level: place_groups (direct), stage_groups / run_staged / fetch, the per-wave fallback, score_assign with dense rows
and top-K keys on both selection kernels, replicated world 2 / 4 contexts, the all-gather scheme, and
place_groups_ranked.  A hand-built case puts nodes free at L but blocked at L - 4 first in the dense rows of groups
at levels 6 and 7, so a level read with two bits in either row table changes the ranked alternates.  Then ragged N at
level 7, hostname keys at a million nodes with the only usable node last in the
background order, and gids at both ends of int32."""
import os
import subprocess
import sys

import numpy as np
import pytest

import levels_limits_cases as C
import levels_oracle as lo
import levels_view as lvw
from oracle import placer as oracle_placer
from rbg_b200 import synth
from rbg_b200.blob import BlobBuilder, Group, GroupsBuilder, ROLE_EXCLUSIVE, STEP_EXCLUSIVE, Step
from rbg_b200.engine import RbgTopoError
from test_gpu_levels_place import _gather, assert_fleet, check_ranked, engine, staged
from test_gpu_steps_limits import FAST_SMEM_MAX, fast_smem

pytestmark = pytest.mark.gpu

ELIMIT = -6


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def install(eng, c):
    eng.set_exclusive_levels(c.lv[1:], c.occ, level_n_domains=c.nd[1:])
    owner = lo.derive_level_owner_fast(c.lv, c.occ)
    got = eng.read_snapshot("level_owner")
    bad = np.argwhere(got != owner)
    assert len(bad) == 0, (len(bad), bad[:4].tolist(), [(int(got[L, v]), int(owner[L, v])) for L, v in bad[:4]])
    return owner


def check_fleet(eng, c, owner, n_alt=8):
    exp, views = lvw.expected_fleet(c.topo, c.lv, owner, c.nd, c.gblob)
    assert_fleet(eng.place_groups(c.gblob), exp, c.gblob, "direct")
    assert_fleet(staged(eng, c.gblob), exp, c.gblob, "staged", staged=True)
    if n_alt:
        check_ranked(eng, c.gblob, views, n_alt)
    return exp


def view_step(c, owner, st):
    """The step on its group's level view (level 0, fixed domain 2d) and the oracle's result there."""
    gids = [st.gid] + ([int(c.gblob[8 + 12 * g]) for g in range(int(c.gblob[2]))] if c.gblob is not None else [])
    view = lvw.level_view(c.topo, c.lv, owner, c.nd, st.level, st.gid, lo.unused_gid(gids))
    vst = Step(**{**st.__dict__, "fixed_domain": 2 * st.fixed_domain if st.fixed_domain >= 0 else -1, "level": 0})
    ref = oracle_placer.place(view, BlobBuilder().add(vst).build(), want_matrix=True, want_topk=True)
    assert ref["rc"] == 0
    return ref


def check_steps(eng, c, owner, steps):
    """One batch of all the steps: score_assign, and stage / run_staged with every dense row and top-K key list."""
    refs = [view_step(c, owner, st) for st in steps]
    bb = BlobBuilder()
    for st in steps:
        bb.add(st)
    blob = bb.build()
    ea = np.concatenate([r["assign"] for r in refs])
    es = np.concatenate([r["status"] for r in refs])
    ed = [x // 2 if x >= 0 else -1 for r in refs for x in r["domain"]]
    a, s, d = eng.score_assign(blob)
    assert np.array_equal(a, ea) and np.array_equal(s, es) and list(d) == ed
    h = eng.stage(blob)
    try:
        eng.run_staged(h, 1)
        a, s, d = eng.fetch(h)
        assert np.array_equal(a, ea) and np.array_equal(s, es) and list(d) == ed
        row = rr = 0
        for i, (st, ref) in enumerate(zip(steps, refs)):
            for k in range(ref["matrix"].shape[0]):
                got = eng.read_scores(h, row + k).view(np.uint32)
                assert np.array_equal(got, ref["matrix"][k].view(np.uint32)), ("row", i, k)
            for p in range(len(st.roles)):
                assert np.array_equal(eng.read_topk(h, rr + p), ref["topk"][p]), ("topk", i, p)
            row += ref["matrix"].shape[0]
            rr += len(st.roles)
    finally:
        eng.release(h)


# ---------------------------------------------------------------- derivation
def test_derivation_past_one_grid_stride():
    c = C.derivation()
    f = C.derivation_facts(c, sm_count=sm_count())
    assert f["phase0"] >= 2 and f["phase1"] >= 2 and f["phase2"] >= 2, f
    eng = engine(c.topo)
    try:
        owner = install(eng, c)
        assert C.derivation_facts(c, owner)["contention_blocked"]
        # an occupancy-only refresh with the records in another order derives the same owners
        perm = np.random.default_rng(0).permutation(len(c.occ))
        eng.set_exclusive_levels(None, c.occ[perm])
        assert np.array_equal(eng.read_snapshot("level_owner"), owner)
    finally:
        eng.close()


def test_partition_reinstalls_never_show_stale_entries():
    topo, seq = C.reinstalls()
    eng = engine(topo)
    try:
        rows, nd = None, None
        for lvl, occ, lnd in seq:
            if lvl is not None:
                rows, nd = lvl, lnd
                eng.set_exclusive_levels(rows, occ, level_n_domains=nd)
            else:
                eng.set_exclusive_levels(None, occ)
            lv = np.vstack([topo.domain[None], rows])
            owner = lo.derive_level_owner_fast(lv, occ)
            assert np.array_equal(eng.read_snapshot("level_owner"), owner), (len(rows), len(occ))
        # the last partitions place groups at levels 1, 4 and 7
        groups = [Group(gid=55 + k, roles=[(0, 3, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE, level=L)
                  for k, L in enumerate((1, 4, 7))]
        c = C.LevelsCase(topo, lv, [len(topo.domain_owner)] + list(nd), occ, gblob=C.build_groups(groups))
        check_fleet(eng, c, owner, n_alt=0)
    finally:
        eng.close()


# ---------------------------------------------------------------- keys 4..7
@pytest.mark.parametrize("seed,n,kind,scarce", C.KEYS47)
def test_keys_4_to_7_match_the_oracle(seed, n, kind, scarce):
    """place_groups (direct), the staged plan and place_groups_ranked with every group at level 4..7, then an
    occupancy-only refresh and a capacity update between calls."""
    c = C.keys47(seed, n, kind, scarce)
    eng = engine(c.topo, chunk_nodes=128)
    try:
        owner = install(eng, c)
        check_fleet(eng, c, owner)
        occ2 = c.occ[::2]
        eng.set_exclusive_levels(None, occ2)
        free2 = np.maximum(c.topo.free - (np.arange(n) % 3 == 0), 0).astype(np.int32)
        eng.update_nodes(free=free2)
        topo2 = synth.Topology(c.topo.row_ptr, c.topo.col_idx, c.topo.edge_w, free2, c.topo.domain,
                               c.topo.domain_owner)
        exp2, _ = lvw.expected_fleet(topo2, c.lv, lo.derive_level_owner_fast(c.lv, occ2), c.nd, c.gblob)
        assert_fleet(eng.place_groups(c.gblob), exp2, c.gblob, "direct after refresh")
    finally:
        eng.close()


@pytest.mark.parametrize("seed,n,kind,scarce", C.KEYS47[1:3])
def test_step_batches_at_keys_4_to_7(seed, n, kind, scarce):
    """Word +14 = 4..7: the batch without its heavy step (k_select_assign_fast), then with it (the global list of
    k_select_assign), dense rows via read_scores and keys via read_topk."""
    c = C.keys47(seed, n, kind, scarce)
    steps = C.steps47(c, seed)
    _, small = fast_smem(c.topo, steps[:-1])
    _, big = fast_smem(c.topo, steps)
    assert small <= FAST_SMEM_MAX < big, (small, big)
    eng = engine(c.topo)
    try:
        owner = install(eng, c)
        check_steps(eng, c, owner, steps[:-1])
        check_steps(eng, c, owner, steps)
    finally:
        eng.close()


def test_per_wave_fallback_at_level_6():
    """A 16-role group at level 6 whose table of patched nodes does not fit k_plan_group's shared memory: the plan
    runs one launch per wave (k_plan_group never launches on a fresh context)."""
    c = C.wide47()
    eng = engine(c.topo)
    try:
        owner = install(eng, c)
        exp, _ = lvw.expected_fleet(c.topo, c.lv, owner, c.nd, c.gblob)
        assert_fleet(staged(eng, c.gblob), exp, c.gblob, "staged", staged=True)
        if not os.environ.get("RBGTOPO_VERIFY_PLAN"):
            assert eng.stats()["plan_ctas"] == 0
        assert_fleet(eng.place_groups(c.gblob), exp, c.gblob, "direct")
    finally:
        eng.close()


@pytest.mark.parametrize("world", [2, 4])
def test_replicated_ranks_at_keys_4_to_7(world):
    """world > 1 contexts on one device place through k_plan_group (a fleet whose tables fit its shared memory)."""
    c = C.keys47(*C.KEYS47[1])
    owner = lo.derive_level_owner_fast(c.lv, c.occ)
    exp, _ = lvw.expected_fleet(c.topo, c.lv, owner, c.nd, c.gblob)
    engs = [engine(c.topo, rank=r, world=world, chunk_nodes=128) for r in range(world)]
    try:
        for e in engs:
            install(e, c)
        for r, e in enumerate(engs):
            assert_fleet(e.place_groups(c.gblob), exp, c.gblob, f"rank {r}")
    finally:
        for e in engs:
            e.close()


@pytest.mark.parametrize("world", [2, 4])
def test_all_gather_scheme_at_keys_4_to_7(world):
    """k_shard_select, k_merge's D* and k_greedy with a device-copy exchange: step batches at levels 4..7 and group
    plans wave by wave, every rank's slab of the dense rows."""
    c = C.keys47(*C.KEYS47[1])
    owner = lo.derive_level_owner_fast(c.lv, c.occ)
    steps = C.steps47(c, world)[:-1]
    refs = [view_step(c, owner, st) for st in steps]
    bb = BlobBuilder()
    for st in steps:
        bb.add(st)
    blob = bb.build()
    exp_fleet, _ = lvw.expected_fleet(c.topo, c.lv, owner, c.nd, c.gblob)
    engs = [engine(c.topo, rank=r, world=world) for r in range(world)]
    try:
        for e in engs:
            install(e, c)
        hs = [e.stage(blob) for e in engs]
        allk = _gather([e.shard_score(h) for e, h in zip(engs, hs)])
        m = [e.shard_merge(h, allk.data_ptr()) for e, h in zip(engs, hs)]
        all2 = _gather([(x[1], x[2]) for x in m]) if m[0][0] else None
        for e, h in zip(engs, hs):
            e.shard_assign(h, all2.data_ptr() if all2 is not None else None)
        for r, (e, h) in enumerate(zip(engs, hs)):
            a, s, d = e.fetch(h)
            off = 0
            lo_, hi = e.slab()
            for i, (st, ref) in enumerate(zip(steps, refs)):
                R = st.n_replicas
                rd = ref["domain"][0] // 2 if ref["domain"][0] >= 0 else -1
                assert a[off:off + R].tolist() == ref["assign"].tolist() and int(s[i]) == int(ref["status"][0]), (r, i)
                assert int(d[i]) == rd, (r, i)
                for k in range(R):
                    got = e.read_scores(h, off + k)
                    assert np.array_equal(got.view(np.uint32), ref["matrix"][k, lo_:hi].view(np.uint32)), (r, i, k)
                off += R
            e.release(h)
        hs = [e.stage_groups(c.gblob) for e in engs]
        for w in range(engs[0].shard_waves(hs[0])):
            allk = _gather([e.shard_wave_score(h, w) for e, h in zip(engs, hs)])
            m = [e.shard_wave_merge(h, w, allk.data_ptr()) for e, h in zip(engs, hs)]
            all2 = _gather([(x[1], x[2]) for x in m]) if m[0][0] else None
            for e, h in zip(engs, hs):
                e.shard_wave_assign(h, w, all2.data_ptr() if all2 is not None else None)
        for r, (e, h) in enumerate(zip(engs, hs)):
            assert_fleet(e.fetch(h), exp_fleet, c.gblob, f"all-gather rank {r}", staged=True)
            e.release(h)
    finally:
        for e in engs:
            e.close()


def test_other_paths_in_a_subprocess():
    """The staged path of place_groups, the per-wave plan and the plan self-check (the host-built plan's level bits
    against the device's) read their switches once when the library loads: the keys-4..7 tests again with each set."""
    here = os.path.dirname(os.path.abspath(__file__))
    me = os.path.join(here, "test_gpu_levels_limits.py")
    for env in ("RBGTOPO_NO_DIRECT", "RBGTOPO_PER_WAVE_PLAN", "RBGTOPO_VERIFY_PLAN"):
        r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "gpu",
                            me + "::test_keys_4_to_7_match_the_oracle", me + "::test_step_batches_at_keys_4_to_7",
                            me + "::test_per_wave_fallback_at_level_6", me + "::test_level_split_at_keys_6_and_7"],
                           env={**os.environ, env: "1"}, capture_output=True, text=True, cwd=os.path.dirname(here))
        assert r.returncode == 0, (env, r.stdout[-3000:] + r.stderr[-3000:])


def test_level_split_at_keys_6_and_7():
    """Nodes free at L but blocked at L - 4 lead the dense rows of the groups placed beside them: on the direct path
    they reach place_groups_ranked's alternates through k_group_rtab's row table, on the staged path through
    k_plan_etab's; a level read with two bits there marks them -inf."""
    c = C.level_split()
    eng = engine(c.topo)
    try:
        owner = install(eng, c)
        check_fleet(eng, c, owner)
        got = eng.place_groups_ranked(c.gblob, 8)
        assert set(got[4][:3].ravel().tolist()) >= set(range(17, 24))     # group 50's alternates: 17..23
    finally:
        eng.close()


# ---------------------------------------------------------------- ragged N, a million nodes, gids at the ends
@pytest.mark.parametrize("n", C.RAGGED)
def test_ragged_node_counts_at_level_7(n):
    """The int4 owner loads of the dense-matrix kernels reach into level_stride's padding of level 7."""
    c = C.ragged(n)
    eng = engine(c.topo)
    try:
        owner = install(eng, c)
        check_fleet(eng, c, owner)
        gids = [int(c.gblob[8 + 12 * g]) for g in range(3)]
        steps = [Step(gid=g, roles=[(2, 1, 1, ROLE_EXCLUSIVE), (1, 0, 1, 0)], pair=[[1, 1], [1, 0]],
                      flags=STEP_EXCLUSIVE, level=7, fixed_domain=-1 if k else int(c.lv[7, n - 1]))
                 for k, g in enumerate(gids)]
        check_steps(eng, c, owner, steps)
    finally:
        eng.close()


def test_hostname_keys_at_a_million_nodes():
    """Levels 5 and 7 hostname-like at N = 2^20 + 1, every node but the last blocked: the restricted selection walks
    the whole background order (every emit chunk) to reach the only usable node."""
    c = C.hostname_1m()
    eng = engine(c.topo)
    try:
        owner = install(eng, c)
        assert C.hostname_facts(c, owner)["only_usable_5"]
        v = c.extra["last"]
        exp = check_fleet(eng, c, owner, n_alt=0)
        assert [e[1] for e in exp] == [0, 0, 1, 2]
        assert exp[1][0] == [v] * 32 and exp[2][0][:3] == [v] * 3 and exp[2][0][3:] == [-1] * 5
    finally:
        eng.close()


def test_gids_at_the_ends_of_int32():
    c = C.gid_ends()
    eng = engine(c.topo)
    try:
        owner = install(eng, c)
        assert {0, C.GID_MAX} <= set(np.unique(owner[6]).tolist())
        exp = check_fleet(eng, c, owner)
        assert exp[0][1] == 0 and exp[1][1] == 0
        steps = [Step(gid=g, roles=[(3, 1, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE, level=6)
                 for g in (0, C.GID_MAX, 7)]
        check_steps(eng, c, owner, steps)
    finally:
        eng.close()


# ---------------------------------------------------------------- the domain ceiling
def test_one_domain_past_the_ceiling_is_refused():
    """0x3FFFFFF1 domains over all levels answers RBGTOPO_ELIMIT before anything is allocated, and the context keeps
    placing, with and without installed levels."""
    over, small = C.ceiling(over=1), C.ceiling(over=-(C.MAX_TOTAL_DOMAINS - 64))
    eng = engine(over.topo)
    ok = GroupsBuilder().add(Group(gid=3, roles=[(0, 2, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE)).build()
    try:
        with pytest.raises(RbgTopoError) as ei:
            eng.set_exclusive_levels(over.lv[1:], over.occ, level_n_domains=over.nd[1:])
        assert ei.value.code == ELIMIT
        assert int(eng.place_groups(ok)[1][0]) == 0
        owner = install(eng, small)                    # a small install, then the refused one again: it stays
        with pytest.raises(RbgTopoError) as ei:
            eng.set_exclusive_levels(over.lv[1:], over.occ, level_n_domains=over.nd[1:])
        assert ei.value.code == ELIMIT
        assert np.array_equal(eng.read_snapshot("level_owner"), owner)
        check_fleet(eng, small, owner, n_alt=0)
    finally:
        eng.close()


def test_domain_ceiling():
    """Exactly 0x3FFFFFF0 domains over all levels is accepted (8 GiB of domain tables, k_level_owner's phase 0 past
    2^31 - stride with 64-bit indices)."""
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < 12 << 30:
        pytest.skip(f"the ceiling case needs 8 GiB of domain tables; {free >> 30} GiB free on a shared device")
    c = C.ceiling()
    assert c.total_domains == C.MAX_TOTAL_DOMAINS
    eng = engine(c.topo)
    try:
        owner = install(eng, c)
        # node 0 is the only member of level 1's last domain and only gid 9 holds it: all four replicas land there
        # (the level view of the oracle would need an owner map of 2^31 entries)
        assert int(owner[1, 0]) == 9
        a, s, d = eng.place_groups(c.gblob)
        assert a.tolist() == [0] * 4 and int(s[0]) == 0 and int(d[0]) == c.nd[1] - 1
    finally:
        eng.close()
