"""CPU: the oracle of ranked alternates for leader-worker pods (tests/lw_alternates_oracle.py, DESIGN.md §3.12).
With one pod per replica and no co-location it is the oracle of ranked placement (§3.10); on generated fleets with
mixed S and C its lists satisfy the rule read as invariants; hand-built cases give known answers.  HAND_CASES is also
run on the device by tests/test_gpu_lw_alternates.py."""
import numpy as np
import pytest

import groups_gen as gg
import lw_oracle as lw
from alternates_oracle import run_fleet_ranked
from lw_alternates_oracle import groups_of, run_lw_ranked, run_lw_rows
from oracle import wave_loop
from rbg_b200 import synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, STEP_GANG, Group, GroupsBuilder


def build(groups):
    gb = GroupsBuilder()
    for g in groups:
        gb.add(g)
    return gb.build()


@pytest.mark.parametrize("seed,n,scarce,excl", gg.CASES)
def test_one_pod_per_replica_is_ranked_placement(seed, n, scarce, excl):
    case = gg.make_case(seed, n, scarce=scarce, exclusive=excl)
    rp = lw.role_pods_for(case.blob, lambda g, r: (1, -1))
    for F in (0, 3, 8):
        got = run_lw_ranked(case.topo, case.blob, rp, F)
        exp = run_fleet_ranked(case.topo, wave_loop.groups_from_blob(case.blob), F)
        for x, y in zip(got, exp):
            assert x.dtype == y.dtype and x.tobytes() == y.tobytes()


def _key_gt(row, a, b):
    return row[a] > row[b] or (row[a] == row[b] and a < b)


@pytest.mark.parametrize("seed,n", [(1, 33), (2, 130), (4, 130), (5, 2049)])
def test_invariants_on_generated_fleets_with_mixed_s_and_c(seed, n):
    """Every alternate is a candidate, the lists are strictly descending in key(score, node), and no candidate that
    outranks the last alternate (or any candidate, when the list has free slots) is left out."""
    case = gg.make_case(seed, n, scarce=seed % 2 == 0, exclusive=True)
    topo, gblob = case.topo, case.blob
    dom = [topo.domain, (np.arange(n) // 4).astype(np.int32)]
    rp = lw.role_pods_for(gblob, lambda g, r: ((2, 1, 3, 4)[(g + r) % 4], (0, -1, 1)[(2 * g + r) % 3]))
    rows = run_lw_rows(topo, gblob, rp, level_domain=dom)[3]
    F = 4
    a, s, d, sc, an, asc = run_lw_ranked(topo, gblob, rp, F, level_domain=dom)
    free = topo.free.astype(np.int64)
    checked = 0
    for g, X in enumerate(groups_of(gblob, rp)):
        pods = slice(X.pod0, X.pod0 + X.n_pods)
        if s[g] == 2:
            assert (a[pods] < 0).all() and np.isneginf(sc[pods]).all() and (an[pods] < 0).all()
            continue
        used = np.zeros(n, np.int64)
        for ri in range(X.q):
            first = X.pod0 + X.first_pod[ri]
            for node in a[first:first + X.pending[ri] * X.S[ri]]:
                if node >= 0:
                    used[node] += X.demand[ri]
        for w, wave in enumerate(X.waves):
            for p, (ri, first, reps) in enumerate(wave):
                base = X.pod0 + X.first_pod[ri] + first * X.S[ri]
                for pod in range(base, base + reps * X.S[ri]):
                    node = int(a[pod])
                    if node < 0:
                        assert np.isneginf(sc[pod]) and (an[pod] < 0).all()
                        continue
                    row = rows[(g, w, p)]
                    assert sc[pod] == row[node]

                    def cand(m):
                        return (row[m] != -np.inf and m != node and free[m] - used[m] >= X.demand[ri]
                                and (not (X.flags & STEP_EXCLUSIVE and X.rflags[ri] & ROLE_EXCLUSIVE)
                                     or topo.domain[m] == d[g])
                                and (X.C[ri] < 0 or dom[X.C[ri]][m] == dom[X.C[ri]][node]))
                    alts = [int(m) for m in an[pod] if m >= 0]
                    assert (an[pod][len(alts):] == -1).all() and np.isneginf(asc[pod][len(alts):]).all()
                    assert all(cand(m) and asc[pod][k] == row[m] for k, m in enumerate(alts))
                    assert all(_key_gt(row, alts[k], alts[k + 1]) for k in range(len(alts) - 1))
                    for m in range(n):
                        if cand(m) and m not in alts:
                            assert len(alts) == F and _key_gt(row, alts[-1], m), (g, pod, m, alts)
                    checked += len(alts)
    assert checked > 0


# ---- hand-built cases: name -> () -> dict(topo, blob, rp, n_alt, levels, level_domain, expect(outputs))

def _flat(n, free=1):
    topo = synth.make_topology(n, seed=11, tiers=2, max_free=2)
    topo.domain_owner = np.full(int(topo.domain.max()) + 1, -1, np.int32)
    topo.free[:] = free
    return topo


def _colocated_alternate_stays_in_domain():
    """A replica of 2 pods co-located at level 0 (domains of 4 nodes, one node of each with no room): its domain
    keeps one free node, which is its only alternate although nodes of other domains outrank it."""
    n = 32
    topo = _flat(n)
    topo.domain = (np.arange(n) // 4).astype(np.int32)
    topo.domain_owner = np.full(8, -1, np.int32)
    topo.free[::4] = 0
    blob = build([Group(gid=1, roles=[(0, 1, 1, 0)], pair=[[1]])])

    def expect(out):
        a, s, d, sc, an, asc = out
        # the replica takes nodes 15 and 13 of domain 3; its free node 14 (27 000) is the alternate of both pods,
        # while nodes 17, 19 and 22 of other domains (27 400) have room and outrank it
        assert a.tolist() == [15, 13] and an.tolist() == [[14, -1, -1]] * 2
        assert asc[:, 0].tolist() == [27000.0] * 2 and sc.tolist() == [27600.0, 27200.0]
    return dict(topo=topo, blob=blob, rp=[(2, 0)], n_alt=3, expect=expect)


def _hostname_level_has_no_alternates():
    n = 16
    topo = _flat(n, free=2)
    levels = [np.arange(n, dtype=np.int32)]
    blob = build([Group(gid=1, roles=[(0, 2, 1, 0)], pair=[[1]])])

    def expect(out):
        a, s, d, sc, an, asc = out
        assert (a >= 0).all() and np.isfinite(sc).all()
        assert (an == -1).all() and np.isneginf(asc).all()
        assert all(a[2 * r] == a[2 * r + 1] for r in range(2))   # both pods of a replica on one host
    return dict(topo=topo, blob=blob, rp=[(2, 1)], n_alt=4, levels=levels, level_domain=[topo.domain, levels[0]],
                expect=expect)


def _node_full_from_sibling_pods_is_skipped():
    """Roles a (S = 2) and b (S = 1) of one wave with equal rows: a takes the two best nodes, which its own pods
    fill; b's pod takes the third, and its alternates start at the fourth."""
    n = 16
    topo = _flat(n)
    blob = build([Group(gid=1, roles=[(0, 1, 1, 0), (0, 1, 1, 0)], pair=[[1, 1], [1, 1]], anchors=[(5, 0, 1)])])

    def expect(out):
        a, s, d, sc, an, asc = out
        assert s.tolist() == [0] and len(set(a.tolist())) == 3
        assert not set(an[2].tolist()) & set(a[:2].tolist())
        assert sc[2] <= min(sc[0], sc[1]) and asc[2][0] <= sc[2]   # a's nodes outrank every alternate of b
    return dict(topo=topo, blob=blob, rp=[(2, -1), (1, -1)], n_alt=4, expect=expect)


def _opted_out_role_leaves_the_exclusive_domain():
    """Exclusive group at level 0 (domains of 4); role b is opted out and co-located at level 1, whose domains (pairs
    of nodes 8 apart) cross the level-0 domains: b's alternates leave domain[g] but stay in b's level-1 domain."""
    n = 16
    topo = _flat(n, free=2)
    topo.domain = (np.arange(n) // 4).astype(np.int32)
    topo.domain_owner = np.full(4, -1, np.int32)
    levels = [(np.arange(n) % 8).astype(np.int32)]
    blob = build([Group(gid=1, roles=[(0, 1, 1, ROLE_EXCLUSIVE), (0, 1, 1, 0)], pair=[[1, 1], [1, 1]],
                        flags=STEP_EXCLUSIVE)])

    def expect(out):
        a, s, d, sc, an, asc = out
        assert d[0] >= 0 and (a >= 0).all()
        assert all(topo.domain[m] == d[0] for m in an[0] if m >= 0)           # participating: inside domain[g]
        b = [int(m) for m in an[1] if m >= 0]
        assert b and all(levels[0][m] == levels[0][a[1]] for m in b)
        assert any(topo.domain[m] != d[0] for m in b)
    return dict(topo=topo, blob=blob, rp=[(1, -1), (1, 1)], n_alt=4, levels=levels,
                level_domain=[topo.domain, levels[0]], expect=expect)


def _gang_failed_group():
    n = 8
    topo = _flat(n)
    blob = build([Group(gid=1, roles=[(0, 1, 1, 0), (1, 2, 1, 0)], pair=[[1, 1], [1, 1]], flags=STEP_GANG),
                  Group(gid=2, roles=[(0, 1, 1, 0)], pair=[[1]])])

    def expect(out):
        a, s, d, sc, an, asc = out
        assert s.tolist() == [2, 0]
        assert (a[:10] == -1).all() and np.isneginf(sc[:10]).all() and (an[:10] == -1).all()
        assert (a[10:] >= 0).all() and (an[10:] >= 0).any()
    return dict(topo=topo, blob=blob, rp=[(2, -1), (4, -1), (2, -1)], n_alt=2, expect=expect)


HAND_CASES = {
    "colocated_alternate_stays_in_domain": _colocated_alternate_stays_in_domain,
    "hostname_level_has_no_alternates": _hostname_level_has_no_alternates,
    "node_full_from_sibling_pods_is_skipped": _node_full_from_sibling_pods_is_skipped,
    "opted_out_role_leaves_the_exclusive_domain": _opted_out_role_leaves_the_exclusive_domain,
    "gang_failed_group": _gang_failed_group,
}


@pytest.mark.parametrize("name", sorted(HAND_CASES))
def test_hand_built_known_answers(name):
    c = HAND_CASES[name]()
    c["expect"](run_lw_ranked(c["topo"], c["blob"], c["rp"], c["n_alt"], level_domain=c.get("level_domain")))
