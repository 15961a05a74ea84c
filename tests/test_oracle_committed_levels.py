"""CPU: the committed oracle at exclusive levels (DESIGN.md §3.8 / §3.9,
committed_levels_oracle.run_fleet_committed_levels).
Hand-built known answers on 6 nodes, equality with run_fleet_committed for batches at level 0, and the brute-force
anti-affinity property on generated mixed-level batches."""
import numpy as np
import pytest

import commit_gen as cg
import commit_levels_gen as clg
import levels_oracle as lo
from committed_levels_oracle import group_levels, level_owner, run_fleet_committed_levels
from committed_oracle import result_arrays, run_fleet_committed
from oracle import wave_loop
from rbg_b200 import synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, STEP_GANG, Group

F = lo.FREE
# 6 nodes on a line, capacity 2 each.  Level 0 = NVLink pairs, level 1 = hostname, level 2 = zone (halves),
# level 3 = parity (crosses the zones)
ROW_PTR = np.array([0, 1, 3, 5, 7, 9, 10], np.int32)
COL = np.array([1, 0, 2, 1, 3, 2, 4, 3, 5, 4], np.int32)
W = np.full(10, 100, np.int32)
LV = np.array([[0, 0, 1, 1, 2, 2], [0, 1, 2, 3, 4, 5], [0, 0, 0, 1, 1, 1], [0, 1, 0, 1, 0, 1]], np.int32)
ND = [3, 6, 2, 2]
HOST, ZONE, PARITY = 1, 2, 3


def topo(free=2):
    return synth.Topology(ROW_PTR, COL, W, np.full(6, free, np.int32), LV[0].copy(), np.full(3, F, np.int32))


def grp(gid, n=1, fixed=-1, gang=False, roles=None):
    roles = roles or [(0, n, 1, ROLE_EXCLUSIVE)]
    return Group(gid=gid, roles=roles, pair=np.eye(len(roles), dtype=int).tolist(), anchors=[],
                 flags=STEP_EXCLUSIVE | (STEP_GANG if gang else 0), fixed_domain=fixed)


def run(groups, levels, occ=(), free=2):
    gb = cg.build(groups)
    for g, L in enumerate(levels):
        gb[8 + 12 * g + 10] = L
    owner = lo.derive_level_owner(LV, np.asarray(occ, np.int32).reshape(-1, 3))
    st = run_fleet_committed_levels(topo(free), wave_loop.groups_from_blob(gb), levels, LV, owner, ND)
    return st, result_arrays(st), owner


def nodes_of(st):
    return [x for x in st.assign_in_group_order() if x >= 0]


def alone(group, level, free=2):
    return run([group], [level], free=free)[0][0]


def test_hostname_then_zone_blocks_the_zone_of_the_pod():
    st, _, owner = run([grp(1), grp(2, n=2)], [HOST, ZONE])
    a = nodes_of(st[0])
    assert len(a) == 1
    z = LV[ZONE, a[0]]
    assert alone(grp(2, n=2), ZONE).result()["domain"] == z          # without the pod, gid 2 takes that zone
    assert st[1].result()["domain"] == 1 - z and all(LV[ZONE, m] != z for m in nodes_of(st[1]))
    # owner_g: the pod's zone is gid 1's (P); the hostname it reported only counts at the hostname level (K)
    last = [np.full(nd, F, np.int32) for nd in ND]
    last[HOST][a[0]] = 1
    exp = np.where(LV[ZONE] == z, 1, F)
    exp[a[0]] = 1
    assert level_owner(LV, owner, ND, ZONE, last, [(1, HOST, a[0])]).tolist() == exp.tolist()


def test_zone_then_hostname_blocks_the_whole_zone():
    st, _, _ = run([grp(2, n=2), grp(1)], [ZONE, HOST])
    z = st[0].result()["domain"]
    assert z >= 0 and alone(grp(1), HOST).result()["domain"] in np.nonzero(LV[ZONE] == z)[0]
    (b,) = nodes_of(st[1])
    assert LV[ZONE, b] != z


def test_crossing_partitions():
    """Parity (level 3) crosses the zones: a parity-level group blocks its parity class (K) for a zone-level group,
    and its pods block their zones (P): only nodes of the other parity in the other zone stay."""
    st, _, owner = run([grp(1), grp(2)], [PARITY, ZONE])
    (a,) = nodes_of(st[0])
    p = st[0].result()["domain"]
    assert p == LV[PARITY, a]
    last = [np.full(nd, F, np.int32) for nd in ND]
    last[PARITY][p] = 1
    own = level_owner(LV, owner, ND, ZONE, last, [(1, PARITY, a)])
    free_nodes = [n for n in range(6) if own[n] == F]
    assert free_nodes == [n for n in range(6) if LV[PARITY, n] != p and LV[ZONE, n] != LV[ZONE, a]]
    (b,) = nodes_of(st[1])
    assert b in free_nodes


def test_opted_out_role_pods_block_nothing():
    """Group 1 (hostname level): an opted-out role first, then a participating one.  Only the participating pod's zone
    is gid 1's for the zone-level group."""
    g1 = Group(gid=1, roles=[(0, 1, 1, 0), (1, 1, 1, ROLE_EXCLUSIVE)], pair=[[1, 0], [0, 1]], anchors=[],
               flags=STEP_EXCLUSIVE)
    st, _, owner = run([g1, grp(2)], [HOST, ZONE], free=1)
    out_pod, part_pod = st[0].assign_in_group_order()
    assert out_pod >= 0 and part_pod >= 0
    last = [np.full(nd, F, np.int32) for nd in ND]
    last[HOST][part_pod] = 1
    own = level_owner(LV, owner, ND, ZONE, last, [(1, HOST, part_pod)])
    assert [int(x) for x in own] == [1 if LV[ZONE, n] == LV[ZONE, part_pod] else F for n in range(6)]
    if LV[ZONE, out_pod] != LV[ZONE, part_pod]:
        assert own[out_pod] == F


def test_a_gang_failed_group_claims_nothing():
    """Three replicas of a hostname-level gang group do not fit one node of capacity 2: it fails, and the zone-level
    group after it sees no claim."""
    st, (a, s, d), owner = run([grp(1, n=3, gang=True), grp(2)], [HOST, ZONE])
    assert int(s[0]) == 2 and int(d[0]) == -1
    assert alone(grp(2), ZONE).assign_in_group_order() == st[1].assign_in_group_order()


def test_two_reporters_at_a_level_the_last_wins():
    """gid 11 then gid 12 report zone 0 (fixed); a later gid-11 zone-level group is kept out of zone 0 by gid 12."""
    st, (a, s, d), _ = run([grp(11, fixed=0), grp(12, fixed=0), grp(11)], [ZONE, ZONE, ZONE], free=4)
    assert d.tolist()[:2] == [0, 0] and int(d[2]) == 1
    # without the second reporter gid 11 goes back into its zone
    st2, (_, _, d2), _ = run([grp(11, fixed=0), grp(11)], [ZONE, ZONE], free=4)
    assert int(d2[1]) == 0


def test_records_still_block():
    """A claim never unblocks what the records block: a zone-level record of gid 9 on node 4 keeps zone 1 from every
    other gid, and the hostname-level group 1 reporting a node there does not change that."""
    st, (a, s, d), owner = run([grp(1), grp(2, n=2)], [HOST, ZONE], occ=[(4, 9, ZONE)])
    assert all(LV[ZONE, m] == 0 for m in nodes_of(st[0]) + nodes_of(st[1]))


def _level0_equal(topo_, gb, lv, occ):
    owner = lo.derive_level_owner(lv, occ)
    nd = [len(topo_.domain_owner)] + [int(lv[L].max()) + 1 for L in range(1, len(lv))]
    groups = wave_loop.groups_from_blob(gb)
    new = result_arrays(run_fleet_committed_levels(topo_, groups, group_levels(gb), lv, owner, nd, fast=True))
    old = result_arrays(run_fleet_committed(topo_, groups, owner0=owner[0], fast=True))
    for x, y in zip(new, old):
        assert np.array_equal(x, y)


@pytest.mark.parametrize("i", range(len(cg.cases())), ids=[c.name for c in cg.cases()])
def test_level0_batches_equal_run_fleet_committed(i):
    """commit_gen's cases with records that reproduce their domain-owner map at level 0."""
    case = cg.cases()[i]
    t = case.topo
    occ = np.array([(int(np.nonzero(t.domain == d)[0][0]), int(o), 0) for d, o in enumerate(t.domain_owner)
                    if o >= 0 and (t.domain == d).any()], np.int32).reshape(-1, 3)
    _level0_equal(t, case.blob, np.asarray(t.domain, np.int32)[None, :], occ)


@pytest.mark.parametrize("i", range(len(cg.occupancy_cases())))
def test_level0_occupancy_batches_equal_run_fleet_committed(i):
    case, lv, occ, _ = cg.occupancy_cases()[i]
    _level0_equal(case.topo, case.blob, lv, occ)


LCASES = clg.cases()


@pytest.mark.parametrize("i", [i for i, c in enumerate(LCASES) if c.topo.n <= 2049],
                         ids=[c.name for c in LCASES if c.topo.n <= 2049])
def test_mixed_level_batches_keep_every_anti_affinity_term(i):
    c = LCASES[i]
    a, s, d = clg.expected(c)
    assert clg.violations(c.lv, c.occ, c.blob, a, s) == []
    assert (s != 2).any() or int(c.blob[2]) == 0
