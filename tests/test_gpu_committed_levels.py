"""GPU: committed batches at exclusive levels (DESIGN.md §3.8 / §3.9, RBGTOPO_CFG_COMMIT_LEVELS): assign, status and
domain bit for bit against committed_levels_oracle.run_fleet_committed_levels, 1 <= rounds <= pending groups, and the
reference's anti-affinity terms kept by every placed participating replica; a batch that needs its second round only
because of a claim across levels; level-0 batches equal with and without the flag (outputs and rounds); world 2 and 4;
partitions reinstalled between calls; the error codes of the flag and of the level words."""
import ctypes as C

import numpy as np
import pytest

import commit_gen as cg
import commit_levels_gen as clg
import levels_oracle as lo
from gpu_util import new_engine
from rbg_b200 import _lib, synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, Group, GroupsBuilder
from rbg_b200.engine import RbgTopoError

pytestmark = pytest.mark.gpu

EINVAL, ELIMIT = -1, -6
LCASES = clg.cases()


def pending_groups(gblob):
    return sum(1 for g in range(int(gblob[2])) if int(gblob[8 + 12 * g + 9]) > 0)


def engine(c, **kw):
    eng = new_engine(c.topo, committed_levels=True, **kw)
    eng.set_exclusive_levels(c.lv[1:], c.occ, level_n_domains=c.nd[1:])
    return eng


def check(eng, c):
    got = eng.place_groups_committed(c.blob)
    a, s, d, rounds = got
    ea, es, ed = clg.expected(c)
    assert np.array_equal(a, ea), (c.name, np.nonzero(a != ea)[0][:8])
    assert np.array_equal(s, es), (c.name, np.nonzero(s != es)[0][:8])
    assert np.array_equal(d, ed), (c.name, np.nonzero(d != ed)[0][:8], d[:16], ed[:16])
    n0 = pending_groups(c.blob)
    assert (rounds == 0) if n0 == 0 else (1 <= rounds <= n0), (rounds, n0)
    return got


@pytest.mark.parametrize("i", range(len(LCASES)), ids=[c.name for c in LCASES])
def test_mixed_level_batches_match_the_oracle(i):
    c = LCASES[i]
    eng = engine(c)
    try:
        a, s, d, _ = check(eng, c)
        assert clg.violations(c.lv, c.occ, c.blob, a, s) == []
    finally:
        eng.close()


def two_round_case():
    """Group 0 (gid 1, hostname level) is fixed to node a, deep in the background order; group 1 (gid 2, zone level)
    reads the order's first 32 nodes, takes its head t and reports t's zone, which also holds a.  Group 1 never reads a
    or a's hostname: only the pod claim of group 0 in that zone (read through dreader[(zone, 0)]) re-runs it."""
    from topo_gen import base_ref, key_node, order_ref
    n = 96
    topo = synth.make_topology(n, seed=3, tiers=2, max_free=4)
    topo.free = np.full(n, 4, np.int32)
    topo.domain_owner[:] = -1
    order = key_node(order_ref(base_ref(topo)))
    t, a = int(order[0]), int(order[40])
    zone = np.ones(n, np.int32)
    zone[[t, a]] = 0
    lv = np.stack([topo.domain, np.arange(n), zone]).astype(np.int32)
    nd = [len(topo.domain_owner), n, 2]
    one = dict(roles=[(0, 1, 1, ROLE_EXCLUSIVE)], pair=[[1]], anchors=[], flags=STEP_EXCLUSIVE)
    gb = GroupsBuilder().add(Group(gid=1, fixed_domain=a, level=1, **one)).add(Group(gid=2, level=2, **one)).build()
    return clg.LevelCase("two_rounds", topo, lv, nd, gb, np.zeros((0, 3), np.int32)), t, a


def test_a_claim_across_levels_takes_exactly_two_rounds():
    c, t, a = two_round_case()
    eng = engine(c)
    try:
        got, s, d, rounds = check(eng, c)
        assert got[0] == a and got[1] >= 0 and c.lv[2, got[1]] == 1 and d.tolist() == [a, 1]
        assert rounds == 2
    finally:
        eng.close()


def test_level0_batches_equal_with_and_without_the_flag():
    """Every commit_gen case and occupancy case: same outputs and rounds on a ctx with both flags."""
    for case in cg.cases():
        e0, e1 = new_engine(case.topo), new_engine(case.topo, committed_levels=True)
        try:
            r0, r1 = e0.place_groups_committed(case.blob), e1.place_groups_committed(case.blob)
            assert all(np.array_equal(x, y) for x, y in zip(r0[:3], r1[:3])) and r0[3] == r1[3], case.name
        finally:
            e0.close()
            e1.close()
    for case, lv, occ, _ in cg.occupancy_cases():
        e0, e1 = new_engine(case.topo), new_engine(case.topo, committed_levels=True)
        try:
            for e in (e0, e1):
                e.set_exclusive_levels(lv[1:], occ)
            r0, r1 = e0.place_groups_committed(case.blob), e1.place_groups_committed(case.blob)
            assert all(np.array_equal(x, y) for x, y in zip(r0[:3], r1[:3])) and r0[3] == r1[3], case.name
        finally:
            e0.close()
            e1.close()


@pytest.mark.parametrize("world", [2, 4])
def test_world_contexts_equal_world_1(world):
    for c in [x for x in LCASES if x.topo.n in (130, 2049)][:3]:
        e1 = engine(c)
        try:
            ref = check(e1, c)
        finally:
            e1.close()
        engs = [engine(c, rank=r, world=world) for r in range(world)]
        try:
            for r, e in enumerate(engs):
                got = e.place_groups_committed(c.blob)
                assert all(np.array_equal(x, y) for x, y in zip(got[:3], ref[:3])) and got[3] == ref[3], (c.name, r)
        finally:
            for e in engs:
                e.close()


def test_partitions_reinstalled_between_calls():
    """One ctx, two installs with different domain counts per level (and different records): each call matches the
    oracle on the partitions installed at the time."""
    base = cg.domains(300, 130)
    c1 = clg.with_levels(base, 301, "mixed")
    c2 = clg.with_levels(base, 302, "random")
    assert c1.nd != c2.nd
    eng = engine(c1)
    try:
        check(eng, c1)
        eng.set_exclusive_levels(c2.lv[1:], c2.occ, level_n_domains=c2.nd[1:])
        check(eng, c2)
        eng.set_exclusive_levels(c1.lv[1:], c1.occ, level_n_domains=c1.nd[1:])
        check(eng, c1)
    finally:
        eng.close()


def _rc(fn, *a):
    try:
        fn(*a)
        return 0
    except RbgTopoError as e:
        return e.code


def test_flags_and_errors_leave_the_ctx_usable():
    lib = _lib.load()
    for flags, rc in ((2, EINVAL), (4, EINVAL), (3, 0)):
        h = C.c_void_p()
        assert lib.rbgtopo_create(C.byref(_lib.Config(device=0, rank=0, world=1, flags=flags)), C.byref(h)) == rc, flags
        if rc == 0:
            assert lib.rbgtopo_destroy(h) == 0
    c = clg.with_levels(cg.domains(310, 64), 310, "mixed")

    def grp(level, fixed=-1):
        return GroupsBuilder().add(Group(gid=3, roles=[(0, 2, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE,
                                         fixed_domain=fixed, level=level)).build()
    lvl_only = new_engine(c.topo, level_placement=True)
    eng = engine(c)
    try:
        lvl_only.set_exclusive_levels(c.lv[1:], c.occ, level_n_domains=c.nd[1:])
        assert _rc(lvl_only.place_groups_committed, grp(1)) == ELIMIT      # levels, but not committed levels
        assert eng.places_committed_levels and not lvl_only.places_committed_levels
        assert _rc(eng.place_groups_committed, grp(4)) == EINVAL            # above n_levels
        assert _rc(eng.place_groups_committed, grp(1, fixed=c.nd[1])) == EINVAL
        assert _rc(eng.place_groups_committed, grp(2, fixed=1)) == EINVAL   # level 2 of 'mixed' has one domain
        check(eng, c)
        a, s, d, _ = eng.place_groups_committed(grp(1, fixed=c.nd[1] - 1))
        assert int(d[0]) in (-1, c.nd[1] - 1)
        assert _rc(lvl_only.place_groups_committed, c.blob) == ELIMIT
        owner = lo.derive_level_owner(c.lv, c.occ)
        assert np.array_equal(eng.read_snapshot("level_owner"), owner)
    finally:
        eng.close()
        lvl_only.close()
