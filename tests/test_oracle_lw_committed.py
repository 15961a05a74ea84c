"""CPU: the oracle of the committed leader-worker batch (tests/lw_committed_oracle.py, DESIGN.md §3.13) reduces to the
committed batch of one pod per replica and to place_groups_lw's loop, does not look ahead, and keeps the section's
invariants on seeded fleets with S in 1..8 and C in {-1, 0, 1, 2}."""
import numpy as np
import pytest

import commit_gen as cg
import lw_commit_gen as lg
import lw_oracle as lw
from committed_oracle import result_arrays, run_fleet_committed
from lw_committed_oracle import run_lw_committed
from oracle import wave_loop


def ones(gblob):
    return lw.role_pods_for(gblob, lambda g, r: (1, -1))


def committed(topo, gblob, owner0=None):
    return result_arrays(run_fleet_committed(topo, wave_loop.groups_from_blob(gblob), owner0=owner0, fast=True))


def same(x, y):
    return all(np.array_equal(np.asarray(a), np.asarray(b)) for a, b in zip(x, y))


@pytest.mark.parametrize("k", range(len(cg.cases())))
def test_one_pod_per_replica_is_the_committed_batch(k):
    case = cg.cases()[k]
    assert same(run_lw_committed(case.topo, case.blob, ones(case.blob)), committed(case.topo, case.blob)), case.name


@pytest.mark.parametrize("k", range(5))
def test_one_pod_per_replica_is_the_committed_batch_in_occupancy_mode(k):
    case, lv, _, owner0 = cg.occupancy_cases()[k]
    got = run_lw_committed(case.topo, case.blob, ones(case.blob), level_domain=lv, owner0=owner0)
    assert same(got, committed(case.topo, case.blob, owner0)), case.name


def check_invariants(f: lg.Fleet, a, s, d):
    rp = f.role_pods()
    used = np.zeros(f.topo.n, dtype=np.int64)
    off, r0 = 0, 0
    reported = {}
    for g, grp in enumerate(f.groups):
        for ri, role in enumerate(grp.roles):
            S, C = (int(x) for x in rp[r0 + ri])
            for _ in range(role[1]):
                pods = a[off:off + S]
                off += S
                assert (pods >= 0).all() or (pods == -1).all(), (g, ri, pods)
                if (pods >= 0).all():
                    used[pods] += role[2]
                    if C >= 0:
                        assert len(set(f.lv[C][pods].tolist())) == 1, (g, ri, pods)
        r0 += len(grp.roles)
        if s[g] == 2:
            continue
        if d[g] >= 0:
            prev = reported.get(int(d[g]))
            assert prev is None or prev == grp.gid or grp.fixed_domain == d[g], (g, d[g], prev, grp.gid)
            reported[int(d[g])] = grp.gid
    assert off == len(a)
    over = np.nonzero(used > f.topo.free)[0]
    assert len(over) == 0, (over[:8], used[over[:8]], f.topo.free[over[:8]])


@pytest.mark.parametrize("seed,n,scarce", lg.SEEDS)
@pytest.mark.parametrize("levels", [False, True])
def test_invariants(seed, n, scarce, levels):
    f = lg.fleet(seed, n, n_groups=12, scarce=scarce, levels=levels, occupancy=levels)
    owner0 = lg.owner0(f) if levels else None
    a, s, d = run_lw_committed(f.topo, f.blob(), f.role_pods(), level_domain=list(f.lv), owner0=owner0)
    check_invariants(f, a, s, d)


@pytest.mark.parametrize("seed,n,scarce", lg.SEEDS[:4])
def test_group_zero_and_one_group_batches_are_place_groups_lw(seed, n, scarce):
    f = lg.fleet(seed, n, scarce=scarce)
    gb, rp = f.blob(), f.role_pods()
    a, s, d = run_lw_committed(f.topo, gb, rp)
    ea, es, ed = lw.run_lw(f.topo, gb, rp)
    n0 = lw.LwGroup(np.asarray(gb, np.int64), 0, rp[:len(f.groups[0].roles)], 0).n_pods
    assert np.array_equal(a[:n0], ea[:n0]) and s[0] == es[0] and d[0] == ed[0]
    for k in range(len(f.groups)):
        one = lg.Fleet(f.topo, [f.groups[k]], [f.rp[k]], f.lv, f.occ)
        assert same(run_lw_committed(f.topo, one.blob(), one.role_pods()), lw.run_lw(f.topo, one.blob(), one.role_pods()))


@pytest.mark.parametrize("seed,n,scarce", lg.SEEDS[:4])
def test_a_group_does_not_depend_on_the_groups_after_it(seed, n, scarce):
    f = lg.fleet(seed, n, scarce=scarce)
    full = run_lw_committed(f.topo, f.blob(), f.role_pods())
    for k in (1, len(f.groups) // 2):
        head = lg.Fleet(f.topo, f.groups[:k], f.rp[:k], f.lv, f.occ)
        a, s, d = run_lw_committed(f.topo, head.blob(), head.role_pods())
        assert np.array_equal(a, full[0][:len(a)]) and np.array_equal(s, full[1][:k]) and np.array_equal(d, full[2][:k])


def gang_failing_fleet(seed):
    """A fleet with a gang group in the middle whose last role asks for more than the whole snapshot holds."""
    f = lg.fleet(seed, 64, n_groups=8)
    k = 4
    g = f.groups[k]
    g.flags |= lw.STEP_GANG
    g.roles[-1] = (g.roles[-1][0], 1, 32767, g.roles[-1][3])
    return f, k


@pytest.mark.parametrize("seed", [11, 12, 13])
def test_a_gang_failed_group_leaves_the_later_groups_as_if_it_were_absent(seed):
    f, k = gang_failing_fleet(seed)
    a, s, d = run_lw_committed(f.topo, f.blob(), f.role_pods())
    assert s[k] == 2
    g = f.without(k)
    b, t, e = run_lw_committed(g.topo, g.blob(), g.role_pods())
    sizes = [sum(r[1] * sc[0] for r, sc in zip(grp.roles, rp)) for grp, rp in zip(f.groups, f.rp)]
    lo, hi = sum(sizes[:k]), sum(sizes[:k + 1])
    assert (a[lo:hi] == -1).all()
    assert np.array_equal(np.concatenate([a[:lo], a[hi:]]), b)
    assert np.array_equal(np.delete(s, k), t) and np.array_equal(np.delete(d, k), e)
