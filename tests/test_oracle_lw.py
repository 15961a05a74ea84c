"""CPU: the oracle of leader-worker placement (tests/lw_oracle.py, DESIGN.md §3.11).  With one pod per replica and no
co-location it is the oracle's own wave loop (oracle/wave_loop.run_fleet); with multi-pod replicas its results keep
the rules: whole replicas in one level-C domain, no node over free, all or nothing, gang, D*; and on tiny instances
the domain a replica lands in is the best one that holds it, found by trying every domain."""
import numpy as np
import pytest

import groups_gen as gg
import lw_oracle as lw
from oracle import wave_loop
from rbg_b200 import synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, STEP_GANG, Group, GroupsBuilder

SMALL = [c for c in gg.CASES if c[1] <= 130]


@pytest.mark.parametrize("seed,n,scarce,excl", SMALL)
def test_one_pod_per_replica_is_the_wave_loop(seed, n, scarce, excl):
    case = gg.make_case(seed, n, scarce=scarce, exclusive=excl)
    a, s, d = lw.run_lw(case.topo, case.blob, lw.role_pods_for(case.blob, lambda g, r: (1, -1)))
    states, _ = wave_loop.run_fleet(case.topo, wave_loop.groups_from_blob(case.blob))
    exp = [x for st in states for x in st.assign_in_group_order()]
    assert a.tolist() == exp
    assert s.tolist() == [st.result()["status"] for st in states]
    assert d.tolist() == [st.result()["domain"] for st in states]


def racks(n, size=4):
    return (np.arange(n) // size).astype(np.int32)


def check_rules(topo, gblob, rp, level_domain, a, s, d):
    gb = np.asarray(gblob)
    rp = np.asarray(rp).reshape(-1, 2)
    off = r0 = 0
    for g in range(int(gb[2])):
        rec = gb[8 + 12 * g: 20 + 12 * g]
        q = int(rec[3])
        roles = gb[rec[4]:rec[4] + 4 * q].reshape(q, 4)
        used = np.zeros(topo.n, np.int64)
        unplaced = 0
        for r in range(q):
            S, C = (int(x) for x in rp[r0 + r])
            for _ in range(int(roles[r, 1])):
                pods = a[off:off + S]
                off += S
                assert (pods >= 0).all() or (pods < 0).all(), pods     # all or nothing
                if pods[0] < 0:
                    unplaced += 1
                    continue
                if C >= 0:
                    assert len(set(level_domain[C][pods].tolist())) == 1, pods
                if (rec[1] & STEP_EXCLUSIVE) and (roles[r, 3] & ROLE_EXCLUSIVE):
                    assert (topo.domain[pods] == d[g]).all()
                np.add.at(used, pods, int(roles[r, 2]))
        r0 += q
        assert (used <= topo.free).all()                               # no node over free
        if s[g] == 2:
            assert rec[1] & STEP_GANG and (a[off - sum(int(roles[r, 1]) * int(rp[r0 - q + r, 0]) for r in range(q)):off] < 0).all()
        else:
            assert (s[g] == 1) == (unplaced > 0)


@pytest.mark.parametrize("seed", range(12))
def test_multi_pod_replicas_keep_the_rules(seed):
    n = (33, 130, 64)[seed % 3]
    case = gg.make_case(seed, n, scarce=seed % 2 == 0, exclusive=seed % 4 != 3)
    rng = np.random.default_rng(seed)
    lv = [case.topo.domain, racks(n)]
    rp = lw.role_pods_for(case.blob, lambda g, r: (int(rng.choice([1, 2, 3, 4])), int(rng.integers(-1, 2))))
    a, s, d = lw.run_lw(case.topo, case.blob, rp, level_domain=lv)
    check_rules(case.topo, case.blob, rp, lv, a, s, d)


def tiny_case(seed):
    rng = np.random.default_rng(seed)
    n = 12
    topo = synth.make_topology(n, seed=seed, tiers=2, max_free=3)
    topo.domain_owner[:] = -1
    demand = int(rng.integers(1, 3))
    S = int(rng.integers(2, 5))
    gb = GroupsBuilder().add(Group(gid=1, roles=[(0, 1, demand, 0)], pair=[[1]],
                                   anchors=[(int(rng.integers(0, n)), 0, 1)])).build()
    return topo, gb, S, demand


@pytest.mark.parametrize("seed", range(40))
def test_the_replica_lands_in_the_best_domain_that_holds_it(seed):
    """One replica of S pods, co-location on racks of 3 nodes: try every rack by placing the pods one after the other
    on its best nodes with room; the oracle picks the rack with the best first pod among those where that succeeds."""
    topo, gb, S, demand = tiny_case(seed)
    dom = (np.arange(topo.n) // 3).astype(np.int32)
    a, s, _ = lw.run_lw(topo, gb, [(S, 0)], level_domain=[dom])
    blob = wave_loop.build_blob([lw.LwGroup(np.asarray(gb, np.int64), 0, np.array([[S, 0]]), 0).step(0)])
    from oracle import placer
    row = placer.place(topo, blob, want_matrix=True, want_topk=False)["matrix"][0]
    best = None
    for d in range(int(dom.max()) + 1):
        room = topo.free.astype(np.int64).copy()
        picks = []
        for _ in range(S):
            m = (dom == d) & (row != -np.inf) & (room >= demand)
            b = lw.best_node(m, row)
            if b < 0:
                break
            room[b] -= demand
            picks.append(b)
        if len(picks) == S and (best is None or lw.better(picks[0], best[1][0], row)):
            best = (d, picks)
    if best is None:
        assert (a < 0).all() and s[0] == 1
    else:
        assert a.tolist() == best[1] and s[0] == 0
