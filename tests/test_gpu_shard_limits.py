"""GPU: node-axis shards at their limits (DESIGN.md §3.17, §3.18), every rank a context on one device and the
all-gather a device concatenation of the ranks' exchange buffers, as in tests/test_gpu_shard_alternates.py.

1. The designed cases of tests/shard_limits_cases.py at the worlds each names, from {2, 3, 4, 5, 8, 16}: every output
   on every rank, fp32 as bits, equals the oracle (not only the world = 1 call) and passes the invariants of
   test_gpu_alternates_limits / test_gpu_lw_limits; the sharded ranked forms at n_alt 0, 1, 3 and 8 (and the case's
   own n_alt), the flagged unranked leader-worker calls.  Cases: the merge lanes at worlds 8 and 16 (every key of
   lane 0 that can win, winners past gathered key 32 only, all nine in one rank, one in each of nine ranks); empty
   first and middle slabs at worlds 3, 4, 5 and 8 with the replica's node at a slab's first and last node and right
   after an empty slab; the four merge layouts of alternates_limits_cases with every OWN kind, shifted to slab_lo =
   2176 and 2304; ties over more than nine nodes across a slab bound, a row of +0.0 over four slabs, fewer candidates
   than n_alt at every n_alt 0..8, an odd compact replica count, jobs not a multiple of the merge's 4 warps, a 32-pod
   job; the slab room bitmap at slab-local bits 0, 31, 32 and len - 1 and just outside the slab, a placement list of
   300 entries over every slab; the patch table of k_lw_assign_repl: hubs of degree 33 and 300, five anchors on one
   hub with an overlapping neighbourhood, an anchor on a consumed node, a consumed record without an anchor (a
   committed batch), a step with an empty table, a wave of P = 8 and P = 1 steps, anchors at node n - 1 for n in
   {31, 33, 8192, 8193}.
2. The existing limit families replayed through the shard entry points at worlds 2, 3 and 8, every rank of every world
   equal and the oracle computed once per case: test_gpu_alternates_limits through shard_place_groups[_committed]_ranked
   (the 1 638 400-node chunk case once, at world 2), test_gpu_lw_limits (without the exactness bounds and the ceiling)
   through RBGTOPO_CFG_LW_SHARDS and shard_place_groups_lw[_committed]_ranked (its two grid-below-steps cases, whose
   replicated scans cost every rank what world 1 costs, at world 2 only), the lw_commit_levels_limits_cases cases on
   flags 15 plus RBGTOPO_CFG_LW_SHARDS.
3. Refusals at worlds 3 and 8 through the raw ABI with sentinel outputs: the enumerated exactness bounds
   (test_gpu_lw_limits.EXACT_CASES, alternates_limits_cases.EXACT) give RBGTOPO_EINEXACT with nothing written and one
   anchor less the calls match the oracle; at world 3, N = 1 638 401 gives RBGTOPO_ELIMIT and N = 1 638 400 places
   as the world = 1 call does."""
import time

import numpy as np
import pytest

import alternates_limits_cases as al
import lw_committed_alternates_oracle as lcao
import lw_oracle as lw
import shard_limits_cases as sc
import test_gpu_alternates_limits as gal
import test_gpu_lw_committed_levels_limits as lcl
import test_gpu_lw_limits as lwl
import test_gpu_lw_shards as lws
import test_gpu_shard_alternates as ash
from rbg_b200 import synth
from rbg_b200.blob import Group

pytestmark = pytest.mark.gpu

EINEXACT, ELIMIT = -4, -6
N_ALTS = (0, 1, 3, 8)
FAMILY_WORLDS = (2, 3, 8)
PEAK = {}


def device_used():
    import torch
    free, total = torch.cuda.mem_get_info()
    return total - free


def shaped(got, F):
    """(assign, status, domain, score, alt_node, alt_score) with the alternates as [replicas][F]."""
    R = len(got[0])
    return (*got[:4], np.asarray(got[4]).reshape(R, F), np.asarray(got[5]).reshape(R, F))


def note_peak(W):
    if W >= 16:
        PEAK[W] = max(PEAK.get(W, 0), device_used())


# ---- 1. the designed cases

@pytest.mark.parametrize("name", sc.ALT_NAMES)
def test_designed_alternates(name):
    _, worlds, n_alts, make = sc.alt_case(name)
    topo, gblob, pre = make()
    exp = pre()
    cexp = gal.committed_oracle(topo, gblob)
    for W in worlds:
        engs = ash.engines(topo, W, lw_shards=True)
        try:
            for F in sorted(set(n_alts) | set(N_ALTS)):
                outs, _ = ash.sharded(engs, gblob, F)
                couts, _ = ash.sharded(engs, gblob, F, committed=True)
                note_peak(W)
                for r, (o, c) in enumerate(zip(outs, couts)):
                    o = shaped(o, F)
                    gal.equal(o, exp, F, (name, W, r))
                    gal.invariants(o[0], o[3], o[4], o[5])
                    c = shaped((*c[:3], *c[4:]), F)
                    gal.equal(c, cexp, F, (name, W, r, "committed"))
                    gal.invariants(c[0], c[3], c[4], c[5])
                    gal.batch_room(topo, gblob, c[0], c[4])
        finally:
            ash.close(engs)


def lw_committed_ranked_oracle(topo, gblob, rp):
    with lw.fast_domains():
        return lcao.run_lw_committed_ranked(topo, gblob, np.asarray(rp, np.int32).reshape(-1, 2), 8)


def check_lw_designed(name, topo, gblob, rp, exp, worlds):
    cexp = sc.committed_oracle(topo, gblob, rp)
    crexp = lw_committed_ranked_oracle(topo, gblob, rp)
    assert all(np.array_equal(x, y) for x, y in zip(crexp[:3], cexp))
    for W in worlds:
        engs = lws.engines(topo, W, lw_shards=True)
        try:
            for r, e in enumerate(engs):
                got = e.place_groups_lw(gblob, rp)
                for x, y in zip(got, exp[:3]):
                    assert np.array_equal(x, y), (name, W, r)
                lwl.invariants(topo, gblob, rp, None, *got)
                a, s, d, rounds = e.place_groups_lw_committed(gblob, rp)
                for x, y in zip((a, s, d), cexp):
                    assert np.array_equal(x, y), (name, W, r, "committed")
                lwl.invariants(topo, gblob, rp, None, a, s, d, committed=True)
            for F in N_ALTS:
                outs, _ = lws.sharded(engs, gblob, rp, F)
                for o in outs:
                    lwl.same(o, exp, F)
            outs, _ = lws.sharded(engs, gblob, rp, 8, committed=True)
            note_peak(W)
            for o in outs:
                lwl.same((*o[:3], *o[4:]), crexp, 8)
        finally:
            ash.close(engs)


@pytest.mark.parametrize("name", sc.LW_CASES)
def test_designed_leader_worker(name):
    topo, gblob, rp, pre = sc.lw_case(name)
    check_lw_designed(name, topo, gblob, rp, pre(), sc.LW_WORLDS)


def test_committed_consumed_record_without_an_anchor():
    topo, gblob, rp, info = sc.committed_consumed_case()
    sc.committed_consumed_pre(topo, gblob, rp, info)
    check_lw_designed("committed_consumed", topo, gblob, rp, sc.lw_ranked_oracle(topo, gblob, rp), sc.LW_WORLDS)


def test_world_16_peak_device_memory(capsys):
    """The lane cases at world 16 again, reporting the device memory in use with their sixteen contexts."""
    base = device_used()
    for name in ("lane0_w16", "nine_ranks_w16"):
        test_designed_alternates(name)
    with capsys.disabled():
        print(f"\nworld 16: peak device memory in use {PEAK[16] / 2**20:.0f} MiB "
              f"({(PEAK[16] - base) / 2**20:.0f} MiB above the {base / 2**20:.0f} MiB in use before)")


# ---- 2. the existing limit families through the shard entry points

class Worlds:
    """An engine-like object over every rank of several worlds (contexts with RBGTOPO_CFG_LW_SHARDS): the ranked
    calls run both shard halves and the merge, the other calls run on every rank; every rank of every world must give
    the same result, which is returned."""

    def __init__(self, topo, setup=None, worlds=FAMILY_WORLDS, **kw):
        self.sets = []
        try:
            for W in worlds:
                self.sets.append(lws.engines(topo, W, setup, lw_shards=True, **kw))
        except BaseException:
            self.close()
            raise

    @staticmethod
    def _one(outs, what):
        for o in outs[1:]:
            if outs[0] is not None:
                lws.same(o, outs[0], what)
        return outs[0]

    def _sharded(self, fn, what):
        return self._one([o for engs in self.sets for o in fn(engs)[0]], what)

    def place_groups_ranked(self, gb, F):
        return self._sharded(lambda engs: ash.sharded(engs, gb, F), "ranked")

    def place_groups_committed_ranked(self, gb, F):
        return self._sharded(lambda engs: ash.sharded(engs, gb, F, committed=True), "committed ranked")

    def place_groups_lw_ranked(self, gb, rp, F):
        return self._sharded(lambda engs: lws.sharded(engs, gb, rp, F), "lw ranked")

    def place_groups_lw_committed_ranked(self, gb, rp, F):
        return self._sharded(lambda engs: lws.sharded(engs, gb, rp, F, committed=True), "lw committed ranked")

    def __getattr__(self, name):
        if name.startswith("_") or name in ("lib", "last_timing"):
            raise AttributeError(name)
        return lambda *a, **k: self._one([getattr(e, name)(*a, **k) for engs in self.sets for e in engs], name)

    def close(self):
        for engs in self.sets:
            ash.close(engs)
        self.sets = []


def levels_setup(lvl):
    return None if lvl is None else (lambda e: e.set_exclusive_levels(lvl[1:], np.zeros((0, 3), np.int32)))


@pytest.fixture
def sharded_engines(monkeypatch):
    """The families' engine() builders replaced by Worlds over worlds 2, 3 and 8."""
    monkeypatch.setattr(lwl, "engine", lambda topo, lvl=None, **kw: Worlds(topo, levels_setup(lvl), **kw))
    monkeypatch.setattr(gal, "engine", lwl.engine)
    monkeypatch.setattr(lcl, "engine", lambda c, **kw: Worlds(
        c.topo, lambda e: e.set_exclusive_levels(c.lv[1:], c.occ, level_n_domains=c.nd[1:]),
        lw_committed_levels=True, **kw))


def family(mod, names):
    """pytest params (test function, kwargs) of every parameter set each named test of mod is parametrized with."""
    out = []
    for name in names:
        fn = getattr(mod, name)
        combos = [{}]
        for m in getattr(fn, "pytestmark", []):
            if m.name != "parametrize":
                continue
            args = [a.strip() for a in m.args[0].split(",")]
            combos = [dict(c, **dict(zip(args, v if len(args) > 1 else (v,)))) for c in combos for v in m.args[1]]
        out += [pytest.param(fn, kw, id="-".join([name[5:]] + [str(v)[:24] for v in kw.values()])) for kw in combos]
    return out


ALT_FAMILY = family(gal, ["test_merge_edges", "test_one_job_of_thirty_two_replicas",
                          "test_ties_over_more_than_nine_nodes_and_a_row_of_zeros",
                          "test_exactly_n_alt_one_more_and_fewer_candidates", "test_colocated_pods_on_the_merge_layouts",
                          "test_room_bitmap_edges", "test_placement_list_longer_than_the_marking_threads",
                          "test_exclusive_group_at_level_one_at_ragged_n", "test_committed_batch_at_all_eight_levels"])
LW_FAMILY = family(lwl, ["test_full_step_of_eight_role_rows_on_a_few_nodes",
                         "test_sizes_that_do_not_divide_32_and_a_zero_pending_role", "test_sixteen_role_groups",
                         "test_room_given_back_by_a_replica_that_fails_part_way", "test_ragged_n_with_the_best_node_last",
                         "test_thirty_two_pods_stacked_on_one_node",
                         "test_seven_levels_colocation_and_exclusive_groups", "test_committed_stale_claims_past_max_free"])
LEVELS_FAMILY = family(lcl, ["test_cases_match_the_oracle_plain_and_ranked"])


@pytest.mark.parametrize("fn,kw", ALT_FAMILY + LW_FAMILY + LEVELS_FAMILY)
def test_limit_families_on_shards(sharded_engines, fn, kw):
    fn(**kw)


@pytest.mark.parametrize("fn,kw", family(lwl, ["test_grid_below_steps_with_colocation",
                                               "test_grid_below_steps_without_colocation"]))
def test_grid_below_steps_at_world_2(monkeypatch, fn, kw):
    """k_lw_assign_repl walking several steps per CTA, each with its own poff slice of the patch tables: at world 2
    only (every rank scans all N nodes per pod, so each world costs what world 1 costs)."""
    monkeypatch.setattr(lwl, "engine", lambda topo, lvl=None, **k: Worlds(topo, levels_setup(lvl), worlds=(2,), **k))
    fn(**kw)


def test_committed_replay_across_chunks_at_world_2():
    """alternates_limits_cases.chunk_case (1 638 400 nodes, three replay chunks) through the sharded committed form."""
    topo, gblob = al.chunk_case()
    exp = gal.committed_oracle(topo, gblob)
    chunks, _ = al.chunk_pre(topo, gblob, exp[0], exp[1])
    assert len(chunks) == 3
    eng = Worlds(topo, worlds=(2,))
    try:
        for F in (8, 1):
            gal.check_committed(eng, topo, gblob, F, exp)
    finally:
        eng.close()


# ---- 3. refusals at worlds 3 and 8

SENT = 12345


def refused(topo, gb, rp, code, worlds=(3, 8)):
    """Every rank: the flagged unranked calls and both sharded ranked local halves return `code`, nothing written."""
    rp = None if rp is None else np.ascontiguousarray(np.asarray(rp, np.int32).reshape(-1))
    for W in worlds:
        engs = lws.engines(topo, W, lw_shards=True)
        try:
            for e in engs:
                for committed in (False, True):
                    assign = np.full(1 << 14, SENT, np.int32)
                    if rp is None:
                        rc, xh, p, nb, _ = ash.raw_local(e, gb, 8, committed, assign)
                    else:
                        rc, rounds = lws.raw_lw(e, gb, rp, committed, assign)
                        assert rc == code and (assign == SENT).all() and rounds == (0 if committed else 9), (W, rc)
                        rc, xh, p, nb, _ = lws.raw_local(e, gb, rp, 8, committed, assign)
                    assert rc == code and (assign == SENT).all() and xh == -7 and not p and nb == -7, (W, rc, xh, nb)
        finally:
            ash.close(engs)


@pytest.mark.parametrize("pair,S,pend,gang", lwl.EXACT_CASES)
def test_leader_worker_exactness_bound(pair, S, pend, gang):
    n = 130
    topo = lwl.free_topo(n, 29, max_free=3)
    topo.free[np.random.default_rng(29).random(n) < 0.6] = 0
    roles, full = lwl.exact_group(pair, pend)
    B = lwl.enumerated_bound(roles[:-1], [r[:-1] for r in full[:-1]], list(S), gang)
    c_at = ((1 << 24) + lwl.gg.wsum_max(topo) + 8000 - 1) // (lwl.gg.wsum_max(topo) + 8000) - max(B)
    rp = [(s, -1) for s in S] + [(1, -1)]
    blob = lambda c: lwl.build([Group(gid=1, roles=roles, pair=full, anchors=[(7, len(pend), c)],
                                      flags=lwl.STEP_GANG if gang else 0)])
    refused(topo, blob(c_at), rp, EINEXACT)
    eng = Worlds(topo, worlds=(3, 8))
    try:
        lwl.run_all(eng, topo, blob(c_at - 1), rp)
    finally:
        eng.close()


@pytest.mark.parametrize("i", range(len(al.EXACT)))
def test_ranked_exactness_bound(i):
    """The committed ranked local half refuses at the bound; the plain one returns the world = 1 call's code."""
    topo, blob, c_at, B = al.exact_case(i)
    e1 = lwl.engine(topo)
    try:
        rc1, _ = lwl.raw(e1, "ranked", blob(c_at))
    finally:
        e1.close()
    assert rc1 in (0, EINEXACT)
    for W in (3, 8):
        engs = ash.engines(topo, W)
        try:
            for e in engs:
                for committed, code in ((True, EINEXACT), (False, rc1)):
                    assign = np.full(1 << 12, SENT, np.int32)
                    rc, xh, p, nb, _ = ash.raw_local(e, blob(c_at), 8, committed, assign)
                    assert rc == code, (W, committed, rc, code)
                    if code:
                        assert (assign == SENT).all() and xh == -7 and not p and nb == -7
        finally:
            ash.close(engs)
    eng = Worlds(topo, worlds=(3, 8))
    try:
        gal.check_committed(eng, topo, blob(c_at - 1), 8, gal.committed_oracle(topo, blob(c_at - 1)))
        gal.check_ranked(eng, topo, blob(c_at - 1), 8, al.ranked(topo, blob(c_at - 1)))
    finally:
        eng.close()


def ring(n):
    """n nodes, each joined to n - 1 and n + 1 (weight 1), free 1 (2 on every 7th), domains of 4 096 nodes."""
    col = np.sort(np.stack([(np.arange(n) - 1) % n, (np.arange(n) + 1) % n], axis=1), axis=1).ravel().astype(np.int32)
    free = np.ones(n, np.int32)
    free[::7] = 2
    return synth.Topology((2 * np.arange(n + 1)).astype(np.int32), col, np.ones(2 * n, np.int32), free,
                          (np.arange(n) // 4096).astype(np.int32), np.full((n + 4095) // 4096, -1, np.int32))


def test_room_bitmap_ceiling_at_world_3():
    t0 = time.perf_counter()
    gb = lwl.build(lwl.ceiling_groups(al.BITMAP_NODES))
    rp = [(4, 0), (2, -1), (3, 0), (32, 0)]
    refused(ring(al.BITMAP_NODES + 1), gb, None, ELIMIT, worlds=(3,))
    refused(ring(al.BITMAP_NODES + 1), gb, rp, ELIMIT, worlds=(3,))
    topo = ring(al.BITMAP_NODES)
    for committed in (False, True):
        ash.check_worlds(topo, gb, n_alts=(8,), committed=committed, worlds=(3,))
        lws.check_worlds(topo, gb, rp, committed=committed, n_alts=(8,), worlds=(3,))
    print(f"ceiling at world 3: {time.perf_counter() - t0:.1f} s")
