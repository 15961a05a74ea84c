"""CPU: the oracle of node eligibility in committed batches (tests/eligible_committed_oracle.py, DESIGN.md §3.20).  With
every mask admitting every class it is the committed leader-worker oracle (and its ranked and levels forms); a one-group
batch is the eligible oracle; a group does not depend on the groups after it; on generated fleets every placed pod and
alternate lies on a node its role admits, no node is over-committed and no exclusivity conflict arises; hand-built
cases, each answered differently without masks or without committing, give known answers.  HAND_CASES is also run on
the device by tests/test_gpu_eligible_committed.py."""
import numpy as np
import pytest

import lw_commit_gen as lg
import lw_commit_levels_gen as lvg
import lw_oracle as lw
from eligible_committed_oracle import (run_eligible_committed, run_eligible_committed_levels,
                                       run_eligible_committed_levels_ranked, run_eligible_committed_ranked)
from eligible_oracle import ALL, admits, full_masks, run_eligible, run_eligible_ranked
from lw_committed_alternates_oracle import run_lw_committed_ranked
from lw_committed_levels_oracle import run_lw_committed_levels, run_lw_committed_levels_ranked
from lw_committed_oracle import groups_of, run_lw_committed
from rbg_b200 import synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, Group
from test_oracle_eligible import random_classes, random_masks
from test_oracle_lw_committed import check_invariants


def same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        x, y = np.asarray(x), np.asarray(y)
        assert x.dtype == y.dtype and x.tobytes() == y.tobytes()


def ones(gblob):
    return lw.role_pods_for(gblob, lambda g, r: (1, -1))


def lv_args(f: lvg.LvFleet):
    return f.lv, f.owner(), f.nd


# ---- the reductions (properties 1-3)

@pytest.mark.parametrize("seed,n,scarce", lg.SEEDS[:4])
@pytest.mark.parametrize("mode", ["map", "occupancy"])
def test_full_masks_are_the_committed_leader_worker_oracle(seed, n, scarce, mode):
    occ = mode == "occupancy"
    f = lg.fleet(seed, n, n_groups=8, scarce=scarce, levels=occ, occupancy=occ)
    gb, rp = f.blob(), f.role_pods()
    kw = dict(level_domain=list(f.lv), owner0=lg.owner0(f)) if occ else {}
    cls = random_classes(n, 5, seed)
    full = full_masks(gb)
    same(run_eligible_committed(f.topo, gb, rp, full, cls, **kw), run_lw_committed(f.topo, gb, rp, **kw))
    same(run_eligible_committed_ranked(f.topo, gb, rp, full, cls, 3, **kw), run_lw_committed_ranked(f.topo, gb, rp, 3, **kw))
    # role_pods None: (S, C) = (1, -1) for every role
    same(run_eligible_committed(f.topo, gb, None, full, cls, **kw), run_lw_committed(f.topo, gb, ones(gb), **kw))


@pytest.mark.parametrize("seed,n,scarce,kind", lvg.SEEDS[1:4])
def test_full_masks_are_the_levels_oracle(seed, n, scarce, kind):
    f = lvg.fleet(seed, n, n_groups=8, scarce=scarce, kind=kind)
    gb, rp = f.blob(), f.role_pods()
    cls = random_classes(n, 3, seed)
    full = full_masks(gb)
    same(run_eligible_committed_levels(f.topo, gb, rp, full, cls, *lv_args(f)),
         run_lw_committed_levels(f.topo, gb, rp, *lv_args(f)))
    same(run_eligible_committed_levels_ranked(f.topo, gb, rp, full, cls, 2, *lv_args(f)),
         run_lw_committed_levels_ranked(f.topo, gb, rp, 2, *lv_args(f)))


@pytest.mark.parametrize("seed,n,scarce", lg.SEEDS[:4])
def test_one_group_batches_are_the_eligible_oracle(seed, n, scarce):
    f = lg.fleet(seed, n, n_groups=6, scarce=scarce)
    cls = random_classes(n, 4, seed)
    for k in range(len(f.groups)):
        one = lg.Fleet(f.topo, [f.groups[k]], [f.rp[k]], f.lv, f.occ)
        gb, rp = one.blob(), one.role_pods()
        masks = random_masks(gb, 4, seed + k)
        same(run_eligible_committed(f.topo, gb, rp, masks, cls), run_eligible(f.topo, gb, rp, masks, cls))
        same(run_eligible_committed_ranked(f.topo, gb, rp, masks, cls, 3), run_eligible_ranked(f.topo, gb, rp, masks, cls, 3))


@pytest.mark.parametrize("seed,n,scarce", lg.SEEDS[:4])
def test_a_group_does_not_depend_on_the_groups_after_it(seed, n, scarce):
    f = lg.fleet(seed, n, n_groups=8, scarce=scarce)
    cls = random_classes(n, 4, seed)
    masks = random_masks(f.blob(), 4, seed)
    full = run_eligible_committed(f.topo, f.blob(), f.role_pods(), masks, cls)
    r0 = 0
    for k in range(1, len(f.groups)):
        r0 += len(f.groups[k - 1].roles)
        head = lg.Fleet(f.topo, f.groups[:k], f.rp[:k], f.lv, f.occ)
        a, s, d = run_eligible_committed(f.topo, head.blob(), head.role_pods(), masks[:r0], cls)
        assert np.array_equal(a, full[0][:len(a)]) and np.array_equal(s, full[1][:k]) and np.array_equal(d, full[2][:k])


# ---- the invariants (property 4) on generated fleets

def check_admitted(gblob, rp, masks, cls, a, alt_node=None):
    checked = 0
    r0 = 0
    for X in groups_of(gblob, rp):
        for ri in range(X.q):
            ok = admits(masks[r0 + ri], cls)
            first = X.pod0 + X.first_pod[ri]
            pods = np.arange(first, first + X.pending[ri] * X.S[ri])
            placed = a[pods][a[pods] >= 0]
            assert ok[placed].all()
            checked += len(placed)
            if alt_node is not None:
                alts = alt_node[pods][alt_node[pods] >= 0]
                assert ok[alts].all()
                checked += len(alts)
        r0 += X.q
    return checked


@pytest.mark.parametrize("seed,n,scarce", lg.SEEDS)
@pytest.mark.parametrize("k", [2, 7, 64])
def test_invariants_at_level_zero(seed, n, scarce, k):
    occ = seed % 2 == 0
    f = lg.fleet(seed, n, n_groups=10, scarce=scarce, levels=occ, occupancy=occ)
    gb, rp = f.blob(), f.role_pods()
    kw = dict(level_domain=list(f.lv), owner0=lg.owner0(f)) if occ else {}
    cls = random_classes(n, k, seed)
    masks = random_masks(gb, k, seed)
    a, s, d, sc, an, asc = run_eligible_committed_ranked(f.topo, gb, rp, masks, cls, 4, **kw)
    same((a, s, d), run_eligible_committed(f.topo, gb, rp, masks, cls, **kw))
    check_admitted(gb, rp, masks, cls, a, an)
    check_invariants(f, a, s, d)


@pytest.mark.parametrize("seed,n,scarce,kind", lvg.SEEDS[1:6])
def test_invariants_at_levels(seed, n, scarce, kind):
    f = lvg.fleet(seed, n, n_groups=10, scarce=scarce, kind=kind)
    gb, rp = f.blob(), f.role_pods()
    cls = random_classes(n, 5, seed)
    masks = random_masks(gb, 5, seed)
    a, s, d, sc, an, asc = run_eligible_committed_levels_ranked(f.topo, gb, rp, masks, cls, 3, *lv_args(f))
    same((a, s, d), run_eligible_committed_levels(f.topo, gb, rp, masks, cls, *lv_args(f)))
    check_admitted(gb, rp, masks, cls, a, an)
    assert lvg.violations(f.lv, f.occ, gb, rp, a, s) == []
    used = np.zeros(n, np.int64)
    for X in groups_of(gb, rp):
        for ri in range(X.q):
            lo = X.pod0 + X.first_pod[ri]
            for node in a[lo:lo + X.pending[ri] * X.S[ri]]:
                if node >= 0:
                    used[node] += X.demand[ri]
    assert (used <= f.topo.free).all()


# ---- hand-built cases: name -> () -> dict(topo, blob, rp, masks, cls, n_alt, expect(outputs), differs(outputs))

def _flat(n, free):
    topo = synth.make_topology(n, seed=11, tiers=2, max_free=2)
    topo.domain = (np.arange(n) // 8).astype(np.int32)
    topo.domain_owner = np.full(n // 8, -1, np.int32)
    topo.free[:] = free
    return topo


def _full_cpu_node():
    """(a) Two CPU-only routers; the unmasked best two nodes are GPU nodes.  The first router takes the last room of
    the best CPU node, so the second moves to another CPU node: not to that full node (the snapshot call) and not to a
    GPU node (unmasked rows)."""
    n = 32
    topo = _flat(n, 1)
    router = lambda gid: Group(gid=gid, roles=[(0, 1, 1, 0)], pair=[[1]])
    blob = lg.build([router(1), router(2)])
    rp = [(1, -1), (1, -1)]
    a0 = run_lw_committed(topo, blob, rp)[0]
    cls = np.zeros(n, np.int32)
    cls[a0] = 1   # the two nodes the unmasked batch picks form the GPU pool
    masks = [0b01, 0b01]
    snap = run_eligible(topo, blob, rp, masks, cls)[0]

    def expect(out):
        a = out[0]
        assert (a >= 0).all() and (cls[a] == 0).all() and a[0] != a[1]
        assert a[1] != snap[1] and a[1] not in a0
    return dict(topo=topo, blob=blob, rp=rp, masks=masks, cls=cls, n_alt=2, expect=expect,
                differs=lambda out: (out[0].tolist() != a0.tolist(), out[0].tolist() != snap.tolist()))


def _map_mode_hand_over():
    """(b) Domain d is owned by gid 9 in the snapshot; an earlier gid-7 group fixes d, so the claim hands d to gid 7,
    and the later gid-7 group, which can only use d, is placed there.  d's best nodes are class 1, which the later
    group's role does not admit: its pods stay on d's admitted nodes."""
    n = 32
    topo = _flat(n, 0)
    d = 1
    topo.domain_owner[d] = 9
    in_d = np.flatnonzero(topo.domain == d)
    topo.free[in_d] = 1
    ex = lambda fixed, cnt: Group(gid=7, roles=[(0, cnt, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE,
                                  fixed_domain=fixed)
    blob = lg.build([ex(d, 1), ex(-1, 2)])
    rp = [(1, -1), (1, -1)]
    a0 = run_lw_committed(topo, blob, rp)[0]
    assert (a0[1:] >= 0).all()   # unmasked, the hand-over gives the later group d's best nodes
    cls = np.zeros(n, np.int32)
    cls[a0[1:]] = 1
    masks = [ALL, 0b01]
    snap = run_eligible(topo, blob, rp, masks, cls)[0]

    def expect(out):
        a, s, dm = out[:3]
        assert (a[1:] >= 0).all() and (cls[a[1:]] == 0).all() and (topo.domain[a[1:]] == d).all() and dm[1] == d
    return dict(topo=topo, blob=blob, rp=rp, masks=masks, cls=cls, n_alt=3, expect=expect,
                differs=lambda out: (out[0].tolist() != a0.tolist(), out[0].tolist() != snap.tolist()))


def _dstar_moves_and_is_avoided():
    """(c) The unmasked D* of the first exclusive group holds no admitted node, so its D* moves; the later group, of
    another gid and with the same mask, avoids the domain the first group actually reports."""
    n = 32
    topo = _flat(n, 2)
    ex = lambda gid: Group(gid=gid, roles=[(0, 2, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE)
    blob = lg.build([ex(1), ex(2)])
    rp = [(1, -1), (1, -1)]
    _, _, d0 = run_lw_committed(topo, blob, rp)
    cls = (topo.domain == d0[0]).astype(np.int32)   # the whole unmasked D* of group 0 is class 1
    masks = [0b01, 0b01]
    unmasked = run_lw_committed(topo, blob, rp)
    snap = run_eligible(topo, blob, rp, masks, cls)

    def expect(out):
        a, s, dm = out[:3]
        assert dm[0] >= 0 and dm[0] != d0[0] and dm[1] >= 0 and dm[1] != dm[0]
        assert (topo.domain[a[:2]] == dm[0]).all() and (topo.domain[a[2:]] == dm[1]).all() and (cls[a] == 0).all()
        assert snap[2][1] == dm[0]   # without committing, group 1 would take group 0's domain
    return dict(topo=topo, blob=blob, rp=rp, masks=masks, cls=cls, n_alt=2, expect=expect,
                differs=lambda out: (out[2].tolist() != unmasked[2].tolist(), out[2].tolist() != snap[2].tolist()))


def _alternate_on_excluded_node():
    """(d) The placements are the unmasked ones (the best nodes are admitted), but the next-best nodes, which the
    unmasked replay rows list as alternates, are class 1: no alternate lies there."""
    n = 32
    topo = _flat(n, 1)
    one = lambda gid: Group(gid=gid, roles=[(0, 1, 1, 0)], pair=[[1]])
    blob = lg.build([one(1), one(2)])
    rp = [(1, -1), (1, -1)]
    ua = run_lw_committed_ranked(topo, blob, rp, 3)
    cls = np.zeros(n, np.int32)
    cls[ua[4][1][:2]] = 1   # the second pod's two best alternates
    cls[ua[0]] = 0
    masks = [ALL, 0b01]

    def expect(out):
        a, an = out[0], out[4]
        assert np.array_equal(a, ua[0]) and (an[1] >= 0).all() and (cls[an[1]] == 0).all()
    return dict(topo=topo, blob=blob, rp=rp, masks=masks, cls=cls, n_alt=3, expect=expect,
                differs=lambda out: (out[4].tolist() != ua[4].tolist(), True))


HAND_CASES = {
    "full_cpu_node": _full_cpu_node,
    "map_mode_hand_over": _map_mode_hand_over,
    "dstar_moves_and_is_avoided": _dstar_moves_and_is_avoided,
    "alternate_on_excluded_node": _alternate_on_excluded_node,
}


@pytest.mark.parametrize("name", sorted(HAND_CASES))
def test_hand_built_known_answers(name):
    c = HAND_CASES[name]()
    out = run_eligible_committed_ranked(c["topo"], c["blob"], c["rp"], c["masks"], c["cls"], c["n_alt"])
    same(out[:3], run_eligible_committed(c["topo"], c["blob"], c["rp"], c["masks"], c["cls"]))
    c["expect"](out)
    assert all(c["differs"](out))   # without masks, and without committing, the answer is another one
