"""CPU: the oracle of ranked alternates for committed batches (tests/committed_alternates_oracle.py, DESIGN.md §3.14).
Its placements are the committed oracle's, a one-group batch is alternates_oracle.run_fleet_ranked, the alternates
obey §3.14 as invariants (room and owner after the whole batch, never the own node, the group's domain, strictly
descending keys), and three known answers: a later group fills a node the snapshot's alternates list, a later
hostname-level group's claim removes an earlier zone-level group's alternate, and a domain handed over in map mode by
a fixed-domain claim leaves the receiving group with finite scores."""
import numpy as np
import pytest

import commit_gen as cg
import committed_alternates_oracle as cao
import levels_oracle as lo
from alternates_oracle import run_fleet_ranked
from committed_oracle import result_arrays, run_fleet_committed
from oracle import wave_loop
from rbg_b200 import synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, Group, GroupsBuilder

FREE = lo.FREE


def small_cases():
    return [cg.gang_frees(), cg.two_reporters(0), cg.domain_move(0)] + [cg.domains(s, 40) for s in range(2)] + \
        [cg.scarce(s, 24) for s in range(4)]


def replicas(gblob):
    """(group, demand, participating) per pending replica in assign order."""
    out = []
    for g, grp in enumerate(wave_loop.groups_from_blob(gblob)):
        for r in grp.roles:
            out += [(g, r.demand, grp.exclusive and r.exclusive)] * r.replicas
    return out


def check_invariants(topo, gblob, res, n_alt, owner_after, dom_of):
    """§3.14 as invariants.  owner_after(g) = own_B,g over the nodes; dom_of(g) = the domain vector of g's level."""
    a, s, d, score, alt, alt_s = res
    groups = wave_loop.groups_from_blob(gblob)
    free = np.asarray(topo.free, np.int64)
    used = np.zeros(len(free), np.int64)
    reps = replicas(gblob)
    for r, (g, dem, _) in enumerate(reps):
        if a[r] >= 0:
            used[a[r]] += dem
    assert (used <= free).all()
    for r, (g, dem, part) in enumerate(reps):
        if a[r] < 0:
            assert score[r] == -np.inf and (alt[r] == -1).all() and (alt_s[r] == -np.inf).all()
            continue
        assert np.isfinite(score[r])
        nodes = [int(x) for x in alt[r] if x >= 0]
        k = len(nodes)
        assert (alt[r][k:] == -1).all() and (alt_s[r][k:] == -np.inf).all()
        assert a[r] not in nodes and len(set(nodes)) == k
        keys = [(float(alt_s[r][i]), -nodes[i]) for i in range(k)]
        assert all(keys[i] > keys[i + 1] for i in range(k - 1)), keys
        for x in nodes:          # moving r to x keeps every node within free[] over the batch
            assert used[x] + dem <= free[x]
        if part:
            own = owner_after(g)
            assert all(dom_of(g)[x] == d[g] and own[x] in (FREE, groups[g].gid) for x in nodes)


def map_owner_after(topo, gblob, d, s):
    own = np.array(topo.domain_owner, np.int32, copy=True)
    for g, grp in enumerate(wave_loop.groups_from_blob(gblob)):
        if grp.exclusive and s[g] != 2 and d[g] >= 0:
            own[d[g]] = grp.gid
    return own[np.asarray(topo.domain)]


@pytest.mark.parametrize("i", range(len(small_cases())))
@pytest.mark.parametrize("n_alt", [0, 1, 8])
def test_placements_are_the_committed_oracles_and_invariants_hold(i, n_alt):
    case = small_cases()[i]
    res = cao.run_fleet_committed_ranked(case.topo, wave_loop.groups_from_blob(case.blob), n_alt)
    ea, es, ed = result_arrays(run_fleet_committed(case.topo, wave_loop.groups_from_blob(case.blob)))
    assert np.array_equal(res[0], ea) and np.array_equal(res[1], es) and np.array_equal(res[2], ed)
    own = map_owner_after(case.topo, case.blob, res[2], res[1])
    check_invariants(case.topo, case.blob, res, n_alt, lambda g: own, lambda g: np.asarray(case.topo.domain))


def test_occupancy_and_levels_invariants():
    case, lv, occ, owner0 = cg.occupancy_cases()[0]
    res = cao.run_fleet_committed_ranked(case.topo, wave_loop.groups_from_blob(case.blob), 4, owner0=owner0)
    ea, es, ed = result_arrays(run_fleet_committed(case.topo, wave_loop.groups_from_blob(case.blob), owner0=owner0))
    assert np.array_equal(res[0], ea) and np.array_equal(res[1], es) and np.array_equal(res[2], ed)
    import commit_levels_gen as clg
    c = clg.cases()[2]
    owner = lo.derive_level_owner(c.lv, c.occ)
    levels = dict(group_levels=clg.group_levels(c.blob), level_domain=c.lv, owner=owner, n_domains=c.nd)
    res = cao.run_fleet_committed_ranked(c.topo, wave_loop.groups_from_blob(c.blob), 8, levels=levels)
    ea, es, ed = clg.expected(c)
    assert np.array_equal(res[0], ea) and np.array_equal(res[1], es) and np.array_equal(res[2], ed)
    gl = clg.group_levels(c.blob)
    check_invariants(c.topo, c.blob, res, 8, lambda g: np.full(c.topo.n, FREE), lambda g: c.lv[gl[g]])
    assert (res[4] >= 0).any()


@pytest.mark.parametrize("i", range(6))
def test_one_group_batch_is_the_ranked_oracle(i):
    case = small_cases()[3 + i % 6]
    for g in wave_loop.groups_from_blob(case.blob)[:3]:
        got = cao.run_fleet_committed_ranked(case.topo, [g], 4)
        exp = run_fleet_ranked(case.topo, [g], 4)
        for x, y in zip(got, exp):
            assert np.array_equal(np.asarray(x).view(np.uint32) if x.dtype == np.float32 else x,
                                  np.asarray(y).view(np.uint32) if y.dtype == np.float32 else y)


def build(groups):
    gb = GroupsBuilder()
    for g in groups:
        gb.add(g)
    return gb.build()


def later_group_fills_case():
    """Nodes of capacity 1, two one-replica groups: the committed batch gives group 1 the node that group 0's
    snapshot alternates list first."""
    topo = synth.make_topology(32, seed=4, tiers=2, max_free=1)
    topo.free = np.ones(32, np.int32)
    topo.domain_owner[:] = -1
    one = dict(roles=[(0, 1, 1, 0)], pair=[[1]], anchors=[(5, 0, 3)], flags=0)
    return topo, [Group(gid=1, **one), Group(gid=2, **one)]


def test_known_answer_a_later_group_fills_a_snapshot_alternate():
    topo, groups = later_group_fills_case()
    gb = build(groups)
    og = wave_loop.groups_from_blob(gb)
    snap = run_fleet_ranked(topo, og[:1], 4)
    got = cao.run_fleet_committed_ranked(topo, og, 4)
    taken = int(got[0][1])
    assert taken == int(snap[4][0][0])                  # group 1 takes group 0's best snapshot alternate
    assert taken not in got[4][0] and got[4][0][0] == snap[4][0][1]


def fixed_handover_case():
    """Map mode: domain D belongs to gid 7 in the snapshot; an idle exclusive group of gid 9 fixed to D claims it, and
    the next gid-9 group is placed there (every other domain has no capacity).  Its rows must not carry the snapshot's
    owner: scores are finite and the alternates lie in D."""
    topo = synth.make_topology(64, seed=8, tiers=2, max_free=2)
    D = int(topo.domain[10])
    topo.domain_owner[:] = -1
    topo.domain_owner[D] = 7
    topo.free = np.where(np.asarray(topo.domain) == D, 2, 0).astype(np.int32)
    idle = Group(gid=9, roles=[(0, 0, 1, ROLE_EXCLUSIVE)], pair=[[1]], anchors=[], flags=STEP_EXCLUSIVE, fixed_domain=D)
    grp = Group(gid=9, roles=[(0, 2, 1, ROLE_EXCLUSIVE)], pair=[[1]], anchors=[], flags=STEP_EXCLUSIVE)
    return topo, [idle, grp], D


def test_known_answer_map_mode_fixed_domain_hand_over():
    topo, groups, D = fixed_handover_case()
    gb = build(groups)
    a, s, d, score, alt, _ = cao.run_fleet_committed_ranked(topo, wave_loop.groups_from_blob(gb), 4)
    assert list(d) == [D, D] and (a >= 0).all() and np.isfinite(score).all()
    nodes = alt[alt >= 0]
    assert len(nodes) and (np.asarray(topo.domain)[nodes] == D).all()


def mixed_level_case(h=None):
    """Levels 0 (the snapshot's domains), 1 (hostname) and 2 (two zones).  Group 0 (gid 1) is exclusive at the zone
    level; group 1 (gid 2) is an idle hostname-level exclusive group fixed to node h.  Returns (topo, lv, nd, blob)."""
    n = 16
    topo = synth.make_topology(n, seed=2, tiers=2, max_free=2)
    topo.domain_owner[:] = -1
    topo.free = np.full(n, 2, np.int32)
    lv = np.stack([topo.domain, np.arange(n), (np.arange(n) >= 8).astype(np.int32)]).astype(np.int32)
    nd = [len(topo.domain_owner), n, 2]
    groups = [Group(gid=1, roles=[(0, 1, 1, ROLE_EXCLUSIVE)], pair=[[1]], anchors=[(3, 0, 2)], flags=STEP_EXCLUSIVE,
                    level=2)]
    if h is not None:
        groups.append(Group(gid=2, roles=[(0, 0, 1, ROLE_EXCLUSIVE)], pair=[[1]], anchors=[], flags=STEP_EXCLUSIVE,
                            fixed_domain=int(h), level=1))
    return topo, lv, nd, build(groups)


def mixed_levels(lv, nd, gb, occ=np.zeros((0, 3), np.int32)):
    import committed_levels_oracle as clo
    return dict(group_levels=clo.group_levels(gb), level_domain=lv, owner=lo.derive_level_owner(lv, occ), n_domains=nd)


def test_known_answer_a_later_hostname_claim_removes_a_zone_alternate():
    topo, lv, nd, gb = mixed_level_case()
    first = cao.run_fleet_committed_ranked(topo, wave_loop.groups_from_blob(gb), 4, levels=mixed_levels(lv, nd, gb))
    h = int(first[4][0][0])
    assert h >= 0
    topo, lv, nd, gb = mixed_level_case(h)
    got = cao.run_fleet_committed_ranked(topo, wave_loop.groups_from_blob(gb), 4, levels=mixed_levels(lv, nd, gb))
    assert got[0][0] == first[0][0] and got[2][1] == h
    assert h not in got[4][0] and list(got[4][0][:3]) == list(first[4][0][1:4])
