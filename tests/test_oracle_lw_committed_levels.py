"""CPU: the oracle of committed leader-worker batches at exclusive levels (tests/lw_committed_levels_oracle.py,
DESIGN.md §3.16): its reductions to the existing oracles, the invariants of the rule, and hand-built known answers,
each with a precondition that the oracle without K, without P or keeping the first reporter gives another result."""
import numpy as np
import pytest

import lw_commit_levels_gen as lvg
import lw_oracle as lw
from committed_levels_oracle import run_fleet_committed_levels
from committed_oracle import result_arrays
from lw_committed_levels_oracle import run_lw_committed_levels, run_lw_committed_levels_ranked
from lw_committed_oracle import groups_of, run_lw_committed
from oracle import wave_loop
from rbg_b200 import synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, STEP_GANG, Group

SEEDS = lvg.SEEDS[:6]


@pytest.mark.parametrize("seed,n,scarce,kind", SEEDS)
def test_level_zero_batches_are_the_committed_lw_oracle(seed, n, scarce, kind):
    f = lvg.fleet(seed, n, scarce=scarce, kind=kind, levels=[0] * 10)
    a, s, d = f.expected()
    ea, es, ed = run_lw_committed(f.topo, f.blob(), f.role_pods(), level_domain=list(f.lv), owner0=f.owner()[0])
    assert np.array_equal(a, ea) and np.array_equal(s, es) and np.array_equal(d, ed)


@pytest.mark.parametrize("seed,n,scarce,kind", SEEDS)
def test_one_pod_per_replica_is_the_committed_levels_oracle(seed, n, scarce, kind):
    f = lvg.fleet(seed, n, scarce=scarce, kind=kind)
    f.rp = [[(1, -1)] * len(rp) for rp in f.rp]
    a, s, d = f.expected()
    blob = f.blob()
    states = run_fleet_committed_levels(f.topo, wave_loop.groups_from_blob(blob), [g.level for g in f.groups], f.lv,
                                        f.owner(), f.nd)
    ea, es, ed = result_arrays(states)
    assert np.array_equal(a, ea) and np.array_equal(s, es) and np.array_equal(d, ed)


@pytest.mark.parametrize("seed,n,scarce,kind", SEEDS)
def test_invariants(seed, n, scarce, kind):
    f = lvg.fleet(seed, n, scarce=scarce, kind=kind)
    gb, rp = f.blob(), f.role_pods()
    a, s, d = f.expected()
    used = np.zeros(f.topo.n, np.int64)
    for g, X in enumerate(groups_of(gb, rp)):
        # a group's results do not depend on the groups after it
        pa, ps, pd = f.sub(range(g + 1)).expected()
        assert np.array_equal(pa, a[:len(pa)]) and ps[g] == s[g] and pd[g] == d[g]
        for ri in range(X.q):
            lo = X.pod0 + X.first_pod[ri]
            for r in range(X.pending[ri]):
                pods = a[lo + r * X.S[ri]:lo + (r + 1) * X.S[ri]]
                assert (pods >= 0).all() or (pods < 0).all()           # all or nothing
                if X.C[ri] >= 0 and (pods >= 0).all():
                    assert len(set(f.lv[X.C[ri]][pods].tolist())) == 1  # one co-location domain
                for m in pods[pods >= 0]:
                    used[m] += X.demand[ri]
    assert (used <= f.topo.free).all()
    assert lvg.violations(f.lv, f.occ, gb, rp, a, s) == []


@pytest.mark.parametrize("seed,n,scarce,kind", SEEDS[:4])
def test_ranked_alternates_break_no_term(seed, n, scarce, kind):
    f = lvg.fleet(seed, n, scarce=scarce, kind=kind)
    gb, rp = f.blob(), f.role_pods()
    a, s, d, score, alt, _ = f.expected_ranked(4)
    assert np.array_equal(a, f.expected()[0])
    G = groups_of(gb, rp)
    for g, X in enumerate(G):
        for ri in range(X.q):
            lo = X.pod0 + X.first_pod[ri]
            for p in range(lo, lo + X.pending[ri] * X.S[ri]):
                for m in alt[p][alt[p] >= 0]:
                    moved = a.copy()
                    moved[p] = m
                    assert lvg.violations(f.lv, f.occ, gb, rp, moved, s) == [], (g, p, m)
                    if X.C[ri] >= 0:
                        assert f.lv[X.C[ri]][m] == f.lv[X.C[ri]][a[p]]


# ---- known answers on 64 nodes: level 1 = hostname, level 2 = zones of 16 nodes
def small():
    topo = synth.make_topology(64, seed=3, tiers=2, max_free=8)
    topo.domain_owner[:] = -1
    topo.free[:] = 4
    lv = np.stack([topo.domain, np.arange(64), np.arange(64) // 16]).astype(np.int32)
    nd = [len(topo.domain_owner), 64, 4]
    return topo, lv, nd


def place(groups, rp, **kw):
    topo, lv, nd = small()
    f = lvg.LvFleet(topo, groups, rp, lv, nd, np.zeros((0, 3), np.int32))
    return f, f.expected(**kw)


def zone(gid, fixed=0, flags=STEP_EXCLUSIVE, rflags=ROLE_EXCLUSIVE, pend=1):
    return Group(gid=gid, roles=[(0, pend, 1, rflags)], pair=[[1]], flags=flags, fixed_domain=fixed, level=2)


def host(gid, fixed=3, flags=STEP_EXCLUSIVE):
    return Group(gid=gid, roles=[(0, 1, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=flags, fixed_domain=fixed, level=1)


def differs(a, b):
    return any(not np.array_equal(x, y) for x, y in zip(a, b))


def test_zone_group_then_hostname_group_needs_k():
    """A zone-keyed group holds zone 0; a later hostname-keyed group fixed to node 3 (in zone 0) may not land there."""
    groups, rp = [zone(1), host(2)], [[(2, -1)], [(1, -1)]]
    f, (a, s, d) = place(groups, rp)
    assert (a[:2] >= 0).all() and (f.lv[2][a[:2]] == 0).all() and a[2] == -1
    assert differs((a, s, d), f.expected(terms=("P",)))


def test_hostname_group_then_zone_group_needs_p():
    """A hostname-keyed pod on node 3 keeps a later zone-keyed group out of zone 0: only its pod (P) says so."""
    groups, rp = [host(2), zone(1)], [[(1, -1)], [(2, -1)]]
    f, (a, s, d) = place(groups, rp)
    assert a[0] == 3 and (a[1:] == -1).all()
    assert differs((a, s, d), f.expected(terms=("K",)))


def test_last_reporter_of_a_zone():
    """Two zone-keyed gids report zone 1 (the second fixed it); a hostname group of the first gid then sees the
    second's claim."""
    groups = [zone(1, fixed=1), zone(2, fixed=1), host(1, fixed=20)]
    rp = [[(1, -1)], [(1, -1)], [(1, -1)]]
    f, (a, s, d) = place(groups, rp)
    assert a[2] == -1
    assert differs((a, s, d), f.expected(reporter="first"))


def test_colocation_at_another_level():
    """A zone-keyed group whose replicas co-locate per host: both pods of a replica on one node of zone 0, and a
    hostname group after it is kept off zone 0 by K."""
    groups, rp = [zone(1, pend=2), host(2)], [[(2, 1)], [(1, -1)]]
    f, (a, s, d) = place(groups, rp)
    assert (a[:4] >= 0).all() and a[0] == a[1] and a[2] == a[3] and (f.lv[2][a[:4]] == 0).all()
    assert a[4] == -1
    assert differs((a, s, d), f.expected(terms=("P",)))


def test_opted_out_role_is_unrestricted():
    """The zone group's opted-out role carries no label: its pods block nothing, and a later hostname group keeps its
    node 3 through P; the participating pods alone would not."""
    groups = [host(2), Group(gid=1, roles=[(0, 1, 1, 0), (0, 1, 1, ROLE_EXCLUSIVE)], pair=[[1, 0], [0, 1]],
                             flags=STEP_EXCLUSIVE, fixed_domain=1, level=2)]
    rp = [[(1, -1)], [(1, -1), (1, -1)]]
    f, (a, s, d) = place(groups, rp)
    assert a[0] == 3 and a[1] >= 0 and a[2] >= 0 and f.lv[2][a[2]] == 1 and s[1] == 0


def test_gang_failure_claims_nothing():
    """A gang-failed zone group (one replica cannot fit) claims no zone: the hostname group after it gets node 3; a
    group that fails without gang would have claimed zone 0."""
    big = zone(1, flags=STEP_EXCLUSIVE | STEP_GANG, pend=3)
    groups, rp = [big, host(2)], [[(32, -1)], [(1, -1)]]
    f, (a, s, d) = place(groups, rp)
    assert s[0] == 2 and (a[:96] == -1).all() and a[96] == 3
    f2, (a2, s2, _) = place([zone(1, pend=3), host(2)], rp)
    assert s2[0] != 2 and a2[96] == -1


def test_ranked_alternates_stay_out_of_later_claims():
    """A zone-keyed group's alternates stay in its zone, and a later hostname group of another gid, kept out of that
    zone by K, takes node 40 of zone 2, which no alternate lists."""
    groups, rp = [zone(1, fixed=1, pend=2), host(2, fixed=40)], [[(1, -1)], [(1, -1)]]
    topo, lv, nd = small()
    f = lvg.LvFleet(topo, groups, rp, lv, nd, np.zeros((0, 3), np.int32))
    a, s, d, score, alt, _ = f.expected_ranked(8)
    assert a[2] == 40 and (lv[2][a[:2]] == 1).all()
    assert 40 not in alt[:2] and (lv[2][alt[:2][alt[:2] >= 0]] == 1).all()
