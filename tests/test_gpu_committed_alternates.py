"""GPU: ranked alternates of committed batches (rbgtopo_place_groups_committed_ranked, DESIGN.md §3.14) bit for bit
against tests/committed_alternates_oracle.py on the same GROUPS blob — assign, status, domain, score, alt_node and
alt_score — on the commit_gen cases (chains, scarce, gang, domains, hub, domain moves, two reporters, extremes), the
occupancy cases and the mixed-level cases on a COMMIT_LEVELS ctx, with n_alt in {0, 1, 8}; equality with
place_groups_committed (rounds included) and, for one-group batches, with place_groups_ranked; NULL status / domain /
rounds; an update_nodes between calls; the exactness bound (RBGTOPO_EINEXACT with nothing written); the error codes
of n_alt, null pointers and world = 2."""
import ctypes as C

import numpy as np
import pytest

import commit_gen as cg
import commit_levels_gen as clg
import committed_alternates_oracle as cao
import levels_oracle as lo
from gpu_util import new_engine
from oracle import wave_loop
from rbg_b200 import _lib, synth
from rbg_b200.blob import Group, GroupsBuilder
from rbg_b200.engine import RbgTopoError

pytestmark = pytest.mark.gpu

EINVAL, ELIMIT, EINEXACT = -1, -6, -4
CASES = cg.cases()
OCC = cg.occupancy_cases()
LCASES = clg.cases()


def bits(x):
    x = np.asarray(x)
    return x.view(np.uint32) if x.dtype == np.float32 else x


def same(got, exp, what=""):
    for i, (x, y) in enumerate(zip(got, exp)):
        assert np.array_equal(bits(x), bits(y)), (what, i, np.nonzero(bits(x) != bits(y))[0][:8])


def check(eng, topo, gblob, n_alt, **oracle_kw):
    got = eng.place_groups_committed_ranked(gblob, n_alt)
    a, s, d, rounds, score, alt, alt_s = got
    exp = cao.run_fleet_committed_ranked(topo, wave_loop.groups_from_blob(gblob), n_alt, fast=True, **oracle_kw)
    same((a, s, d, score, alt, alt_s), exp, "oracle")
    plain = eng.place_groups_committed(gblob)
    same(plain[:3], (a, s, d), "place_groups_committed")
    assert plain[3] == rounds
    return got


@pytest.mark.parametrize("i", range(len(CASES)), ids=[c.name for c in CASES])
def test_commit_gen_cases_match_the_oracle(i):
    case = CASES[i]
    eng = new_engine(case.topo)
    try:
        for n_alt in (0, 1, 8):
            check(eng, case.topo, case.blob, n_alt)
    finally:
        eng.close()


@pytest.mark.parametrize("i", range(len(OCC)))
def test_occupancy_cases_match_the_oracle(i):
    case, lv, occ, owner0 = OCC[i]
    eng = new_engine(case.topo, committed_levels=True)
    try:
        eng.set_exclusive_levels(lv[1:], occ)
        for n_alt in (1, 8):
            check(eng, case.topo, case.blob, n_alt, owner0=owner0)
    finally:
        eng.close()


@pytest.mark.parametrize("i", range(len(LCASES)), ids=[c.name for c in LCASES])
def test_mixed_level_cases_match_the_oracle(i):
    c = LCASES[i]
    eng = new_engine(c.topo, committed_levels=True)
    try:
        eng.set_exclusive_levels(c.lv[1:], c.occ, level_n_domains=c.nd[1:])
        levels = dict(group_levels=clg.group_levels(c.blob), level_domain=c.lv, owner=lo.derive_level_owner(c.lv, c.occ),
                      n_domains=c.nd)
        for n_alt in (0, 8):
            check(eng, c.topo, c.blob, n_alt, levels=levels)
    finally:
        eng.close()


def test_known_answers_on_the_device():
    """The three known answers of tests/test_oracle_committed_alternates.py, placed by the library."""
    from test_oracle_committed_alternates import (build, fixed_handover_case, later_group_fills_case, mixed_level_case,
                                                  mixed_levels)
    topo, groups = later_group_fills_case()
    eng = new_engine(topo)
    try:
        gb = build(groups)
        got = check(eng, topo, gb, 4)
        snap = eng.place_groups_ranked(build(groups[:1]), 4)
        assert got[0][1] == snap[4][0][0] and got[0][1] not in got[5][0]
    finally:
        eng.close()
    topo, groups, D = fixed_handover_case()
    eng = new_engine(topo)
    try:
        got = check(eng, topo, build(groups), 4)
        assert np.isfinite(got[4]).all() and (got[5] >= 0).any()
    finally:
        eng.close()
    topo, lv, nd, gb0 = mixed_level_case()
    eng = new_engine(topo, committed_levels=True)
    try:
        eng.set_exclusive_levels(lv[1:], np.zeros((0, 3), np.int32), level_n_domains=nd[1:])
        first = check(eng, topo, gb0, 4, levels=mixed_levels(lv, nd, gb0))
        h = int(first[5][0][0])
        _, _, _, gb = mixed_level_case(h)
        got = check(eng, topo, gb, 4, levels=mixed_levels(lv, nd, gb))
        assert got[0][0] == first[0][0] and h not in got[5][0]
    finally:
        eng.close()


def test_one_group_batches_equal_place_groups_ranked():
    eng = None
    try:
        for case in [cg.scarce(3, 40), cg.domains(2, 96), cg.table_reads(0)]:
            eng = new_engine(case.topo)
            b = np.asarray(case.blob)
            for g in range(min(int(b[2]), 8)):
                one = GroupsBuilder().add(_group_of(b, g)).build()
                got = eng.place_groups_committed_ranked(one, 8)
                exp = eng.place_groups_ranked(one, 8)
                same(got[:3] + got[4:], exp, f"group {g}")
                assert got[3] == (1 if int(one[4]) > 0 else 0)
            eng.close()
            eng = None
    finally:
        if eng is not None:
            eng.close()


def _group_of(b, i):
    gid, flags, fixed, q, role_off, pair_off, na, anchor_off = (int(x) for x in b[8 + 12 * i:][:8])
    roles = [tuple(int(x) for x in b[role_off + 4 * r:role_off + 4 * r + 4]) for r in range(q)]
    pair = b[pair_off:pair_off + q * q].reshape(q, q).tolist()
    anchors = [tuple(int(x) for x in b[anchor_off + 3 * a:anchor_off + 3 * a + 3]) for a in range(na)]
    return Group(gid=gid, roles=roles, pair=pair, anchors=anchors, flags=flags, fixed_domain=fixed)


def raw_call(eng, gb, n_alt, assign, status, domain, rounds, score, alt, alt_s):
    p = lambda a, t=_lib.i32p: None if a is None else a.ctypes.data_as(t)
    return eng.lib.rbgtopo_place_groups_committed_ranked(
        eng._h, p(gb), len(gb), n_alt, p(assign), p(status), p(domain), None if rounds is None else C.byref(rounds),
        p(score, _lib.f32p), p(alt), p(alt_s, _lib.f32p))


def test_null_outputs_update_nodes_and_error_codes():
    case = cg.scarce(5, 40)
    gb = np.asarray(case.blob, np.int32)
    R = int(gb[4])
    eng = new_engine(case.topo)
    try:
        ref = check(eng, case.topo, gb, 8)
        score, alt, alt_s, assign = (np.empty(R, np.float32), np.empty((R, 8), np.int32), np.empty((R, 8), np.float32),
                                     np.empty(R, np.int32))
        assert raw_call(eng, gb, 8, assign, None, None, None, score, alt, alt_s) == 0
        same((assign, score, alt, alt_s), (ref[0], ref[4], ref[5], ref[6]), "NULL status / domain / rounds")
        assert raw_call(eng, gb, 0, assign, None, None, None, score, None, None) == 0
        same((assign, score), (ref[0], ref[4]), "n_alt 0")
        # codes, nothing written
        for n_alt, args in [(9, (assign, None, None, None, score, alt, alt_s)),
                            (-1, (assign, None, None, None, score, alt, alt_s)),
                            (4, (None, None, None, None, score, alt, alt_s)),
                            (4, (assign, None, None, None, None, alt, alt_s)),
                            (4, (assign, None, None, None, score, None, alt_s))]:
            assert raw_call(eng, gb, n_alt, *args) == EINVAL
        # a refresh between calls
        rng = np.random.default_rng(1)
        free = np.asarray(case.topo.free, np.int32).copy()
        free[rng.choice(len(free), size=len(free) // 3, replace=False)] += 1
        eng.update_nodes(free=free)
        topo2 = synth.Topology(case.topo.row_ptr, case.topo.col_idx, case.topo.edge_w, free, case.topo.domain,
                               case.topo.domain_owner)
        check(eng, topo2, gb, 8)
    finally:
        eng.close()
    engs = [new_engine(case.topo, rank=r, world=2) for r in range(2)]
    try:
        for e in engs:
            with pytest.raises(RbgTopoError) as ex:
                e.place_groups_committed_ranked(gb, 4)
            assert ex.value.code == ELIMIT
    finally:
        for e in engs:
            e.close()


def test_the_exactness_bound_of_the_ranking():
    """A non-gang two-wave group whose anchor weight puts it between the bound place_groups_committed checks and the
    one the ranking needs (unplaced replicas of the first wave raise need in the second): RBGTOPO_EINEXACT before any
    round, nothing written; place_groups_committed accepts it."""
    topo = synth.make_topology(256, seed=3, tiers=2, max_free=2)
    eng = new_engine(topo)
    blob = lambda A: GroupsBuilder().add(Group(gid=1, roles=[(0, 40, 1, 0)], pair=[[1]], anchors=[(7, 0, A)],
                                               flags=0)).build()
    try:
        lo_, hi = 1, 1 << 20        # the largest anchor count place_groups_committed accepts
        while hi - lo_ > 1:
            mid = (lo_ + hi) // 2
            try:
                eng.place_groups_committed(blob(mid))
                lo_ = mid
            except RbgTopoError as e:
                assert e.code == EINEXACT
                hi = mid
        gb = blob(lo_)
        assign = np.full(40, 12345, np.int32)
        score = np.full(40, 7.0, np.float32)
        rounds = C.c_int32(9)
        assert raw_call(eng, gb, 0, assign, None, None, rounds, score, None, None) == EINEXACT
        assert rounds.value == 0 and (assign == 12345).all() and (score == 7.0).all()
        check(eng, topo, GroupsBuilder().add(Group(gid=1, roles=[(0, 40, 1, 0)], pair=[[1]], anchors=[(7, 0, 3)],
                                                   flags=0)).build(), 8)
    finally:
        eng.close()
