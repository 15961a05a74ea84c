"""CPU: the oracle of ranked alternates for committed leader-worker batches (tests/lw_committed_alternates_oracle.py,
DESIGN.md §3.15).  Its placements are the committed leader-worker oracle's; a one-group batch is
lw_alternates_oracle.run_lw_ranked; one pod per replica without co-location is committed_alternates_oracle in map and
occupancy mode; the alternates obey §3.15 as invariants (room after the whole batch, no other gid's claim, the
replica's co-location domain); and three known answers: a later group's pods fill a node the snapshot's alternates
list, a later group of another gid fixed to a domain removes an earlier reporter's alternates there (map mode), and a
better node outside the replica's co-location domain never appears."""
import numpy as np
import pytest

import commit_gen as cg
import committed_alternates_oracle as cao
import lw_commit_gen as lg
import lw_oracle as lw
from committed_oracle import FREE, merge_claims
from lw_alternates_oracle import run_lw_ranked
from lw_committed_alternates_oracle import run_lw_committed_ranked, run_lw_committed_rows
from lw_committed_oracle import run_lw_committed
from oracle import wave_loop
from rbg_b200 import synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, Group


def bits(x):
    x = np.asarray(x)
    return x.view(np.uint32) if x.dtype == np.float32 else x


def same(x, y):
    return all(np.array_equal(bits(a), bits(b)) for a, b in zip(x, y))


def ones(gblob):
    return lw.role_pods_for(gblob, lambda g, r: (1, -1))


def pods_of(f: lg.Fleet):
    """(group, role, demand, C, participating, first pod of the replica) per pod in assign order."""
    out, r0 = [], 0
    rp = f.role_pods()
    for g, grp in enumerate(f.groups):
        excl = bool(grp.flags & STEP_EXCLUSIVE)
        for ri, role in enumerate(grp.roles):
            S, C = (int(x) for x in rp[r0 + ri])
            for _ in range(role[1]):
                first = len(out)
                out += [(g, ri, role[2], C, excl and bool(role[3] & ROLE_EXCLUSIVE), first)] * S
        r0 += len(grp.roles)
    return out


def owner_after(f: lg.Fleet, s, d, owner0=None):
    """own_B over the nodes: the snapshot's level-0 owner with every domain's last reporter in the batch applied."""
    last = np.full(len(f.topo.domain_owner), FREE, np.int32)
    for g, grp in enumerate(f.groups):
        if (grp.flags & STEP_EXCLUSIVE) and s[g] != 2 and d[g] >= 0:
            last[d[g]] = grp.gid
    if owner0 is not None:
        return merge_claims(np.asarray(owner0, np.int32), last[f.topo.domain])
    own = np.array(f.topo.domain_owner, np.int32, copy=True)
    own[last != FREE] = last[last != FREE]
    return own[f.topo.domain]


def check_invariants(f: lg.Fleet, res, owner0=None):
    a, s, d, score, alt, alt_s = res
    free = np.asarray(f.topo.free, np.int64)
    pods = pods_of(f)
    assert len(pods) == len(a)
    used = np.zeros(len(free), np.int64)
    for p, (_, _, dem, _, _, _) in enumerate(pods):
        if a[p] >= 0:
            used[a[p]] += dem
    assert (used <= free).all()
    own = owner_after(f, s, d, owner0)
    listed = 0
    for p, (g, _, dem, C, part, _) in enumerate(pods):
        if a[p] < 0:
            assert score[p] == -np.inf and (alt[p] == -1).all() and (alt_s[p] == -np.inf).all()
            continue
        assert np.isfinite(score[p])
        nodes = [int(x) for x in alt[p] if x >= 0]
        k = len(nodes)
        listed += k
        assert (alt[p][k:] == -1).all() and (alt_s[p][k:] == -np.inf).all()
        assert a[p] not in nodes and len(set(nodes)) == k
        keys = [(float(alt_s[p][i]), -nodes[i]) for i in range(k)]
        assert all(keys[i] > keys[i + 1] for i in range(k - 1)), keys
        for x in nodes:
            assert used[x] + dem <= free[x]                      # moving p to x over-commits no node
            if part:                                             # no other gid's claim in the batch forbids x
                assert f.topo.domain[x] == d[g] and own[x] in (FREE, f.groups[g].gid), (p, x, own[x])
            if C >= 0:                                           # the replica stays co-located
                assert f.lv[C][x] == f.lv[C][a[p]]
    return listed


@pytest.mark.parametrize("seed,n,scarce", lg.SEEDS)
@pytest.mark.parametrize("mode", ["map", "occupancy"])
def test_placements_are_the_committed_oracles_and_invariants_hold(seed, n, scarce, mode):
    occ = mode == "occupancy"
    f = lg.fleet(seed, n, n_groups=10, scarce=scarce, levels=occ, occupancy=occ)
    owner0 = lg.owner0(f) if occ else None
    gb, rp = f.blob(), f.role_pods()
    res = run_lw_committed_ranked(f.topo, gb, rp, 8, level_domain=list(f.lv), owner0=owner0)
    assert same(res[:3], run_lw_committed(f.topo, gb, rp, level_domain=list(f.lv), owner0=owner0))
    check_invariants(f, res, owner0)


@pytest.mark.parametrize("seed,n,scarce", lg.SEEDS[:4])
def test_one_group_batch_is_the_lw_ranked_oracle(seed, n, scarce):
    f = lg.fleet(seed, n, n_groups=6, scarce=scarce)
    for k in range(len(f.groups)):
        one = lg.Fleet(f.topo, [f.groups[k]], [f.rp[k]], f.lv, f.occ)
        assert same(run_lw_committed_ranked(f.topo, one.blob(), one.role_pods(), 4),
                    run_lw_ranked(f.topo, one.blob(), one.role_pods(), 4)), k


@pytest.mark.parametrize("k", [3, 4, 5, 8, 9, 12, 14])
@pytest.mark.parametrize("n_alt", [0, 3])
def test_one_pod_per_replica_is_the_committed_alternates_oracle(k, n_alt):
    case = cg.cases()[k]
    got = run_lw_committed_ranked(case.topo, case.blob, ones(case.blob), n_alt)
    exp = cao.run_fleet_committed_ranked(case.topo, wave_loop.groups_from_blob(case.blob), n_alt)
    assert same(got, exp), case.name


@pytest.mark.parametrize("k", range(5))
def test_one_pod_per_replica_is_the_committed_alternates_oracle_in_occupancy_mode(k):
    case, lv, _, owner0 = cg.occupancy_cases()[k]
    got = run_lw_committed_ranked(case.topo, case.blob, ones(case.blob), 4, level_domain=list(lv), owner0=owner0)
    exp = cao.run_fleet_committed_ranked(case.topo, wave_loop.groups_from_blob(case.blob), 4, owner0=owner0)
    assert same(got, exp), case.name


def unit_topology(n=32, free=1):
    topo = synth.make_topology(n, seed=4, tiers=2, max_free=free)
    topo.free = np.full(n, free, np.int32)
    topo.domain_owner[:] = -1
    return topo


def test_known_answer_a_later_groups_pods_fill_a_snapshot_alternate():
    """Nodes of capacity 1, two groups of one two-pod replica pulled to node 5: the second group's pods take the two
    nodes the first group's place_groups_lw_ranked alternates list first."""
    topo = unit_topology()
    one = dict(roles=[(0, 1, 1, 0)], pair=[[1]], anchors=[(5, 0, 3)], flags=0)
    groups = [Group(gid=1, **one), Group(gid=2, **one)]
    rp = [(2, -1), (2, -1)]
    snap = run_lw_ranked(topo, lg.build(groups[:1]), rp[:1], 4)
    a, _, _, _, alt, _ = run_lw_committed_ranked(topo, lg.build(groups), rp, 4)
    taken = [int(x) for x in a[2:]]
    assert taken == [int(x) for x in snap[4][0][:2]]
    for p in (0, 1):
        assert not set(taken) & set(alt[p].tolist())
        assert list(alt[p][:2]) == list(snap[4][p][2:4])


def test_known_answer_a_later_fixed_domain_claim_removes_an_earlier_reporters_alternates():
    """Map mode: group 0 (gid 1) reports domain D; an idle group of gid 2 fixed to D then claims it, so no node of D
    is -1 or gid 1 for the batch any more and every participating alternate of group 0 goes."""
    topo = unit_topology(free=2)
    first = Group(gid=1, roles=[(0, 1, 1, ROLE_EXCLUSIVE)], pair=[[1]], anchors=[(5, 0, 3)], flags=STEP_EXCLUSIVE)
    alone = run_lw_committed_ranked(topo, lg.build([first]), [(2, 0)], 4)
    D = int(alone[2][0])
    assert D == topo.domain[5] and (alone[4] >= 0).sum() == 8
    idle = Group(gid=2, roles=[(0, 0, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE, fixed_domain=D)
    a, s, d, score, alt, alt_s = run_lw_committed_ranked(topo, lg.build([first, idle]), [(2, 0), (2, 0)], 4)
    assert np.array_equal(a, alone[0]) and list(d) == [D, D] and np.array_equal(bits(score), bits(alone[3]))
    assert (alt == -1).all() and (alt_s == -np.inf).all()


def test_known_answer_a_better_node_outside_the_colocation_domain_never_appears():
    """Anchors on node 5 (3) and node 20 (2), another level-0 domain: the replica of two pods lands in node 5's
    domain, and node 20, which outscores every node left there, is no alternate; without co-location it is."""
    topo = unit_topology()
    grp = Group(gid=1, roles=[(0, 1, 1, 0)], pair=[[1]], anchors=[(5, 0, 3), (20, 0, 2)], flags=0)
    gb = lg.build([grp])
    a, _, _, rows = run_lw_committed_rows(topo, gb, [(2, 0)])
    res = run_lw_committed_ranked(topo, gb, [(2, 0)], 8)
    D = topo.domain[a[0]]
    assert topo.domain[a[1]] == D and topo.domain[20] != D
    row = rows[(0, 0, 0)]
    for p in (0, 1):
        nodes = res[4][p][res[4][p] >= 0]
        assert len(nodes) and (topo.domain[nodes] == D).all() and 20 not in nodes
        assert row[20] > row[nodes].max()
    free = run_lw_committed_ranked(topo, gb, [(2, -1)], 8)
    assert 20 in free[0]
