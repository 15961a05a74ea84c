"""CPU: the oracle of node eligibility (tests/eligible_oracle.py, DESIGN.md §3.19).  With every mask admitting every
class it is the leader-worker oracle and its ranked form; on generated fleets every placed pod and every alternate
lies on a node its role admits and keeps the unmasked row's score; hand-built cases, each of which the unmasked oracle
answers differently, give known answers.  HAND_CASES is also run on the device by tests/test_gpu_eligible.py."""
import numpy as np
import pytest

import groups_gen as gg
import lw_oracle as lw
from eligible_oracle import ALL, admits, full_masks, run_eligible, run_eligible_ranked
from lw_alternates_oracle import groups_of, run_lw_ranked, run_lw_rows
from rbg_b200 import synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, STEP_GANG, Group, GroupsBuilder

SMALL = [c for c in gg.CASES if c[1] <= 130]


def build(groups):
    gb = GroupsBuilder()
    for g in groups:
        gb.add(g)
    return gb.build()


def mixed_pods(gblob):
    return lw.role_pods_for(gblob, lambda g, r: ((2, 1, 3)[(g + r) % 3], (-1, 0)[(g + 2 * r) % 2]))


def random_classes(n, k, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(0, k, n).astype(np.int32)


def random_masks(gblob, k, seed):
    """Per role a mask of one class up to all but one of k classes (all classes when k == 1)."""
    rng = np.random.default_rng(seed + 1000)
    out = []
    for _ in range(len(full_masks(gblob))):
        if k == 1:
            out.append(ALL)
            continue
        keep = rng.choice(k, int(rng.integers(1, k)), replace=False)
        out.append(int(sum(1 << int(c) for c in keep)))
    return np.asarray(out, dtype=np.uint64)


def same(a, b):
    for x, y in zip(a, b):
        assert x.dtype == y.dtype and x.tobytes() == y.tobytes()


@pytest.mark.parametrize("seed,n,scarce,excl", SMALL)
def test_full_masks_are_the_leader_worker_oracle(seed, n, scarce, excl):
    case = gg.make_case(seed, n, scarce=scarce, exclusive=excl)
    cls = random_classes(n, 5, seed)
    full = full_masks(case.blob)
    for rp in (mixed_pods(case.blob), None):
        ref_rp = lw.role_pods_for(case.blob, lambda g, r: (1, -1)) if rp is None else rp
        same(run_eligible(case.topo, case.blob, rp, full, cls), lw.run_lw(case.topo, case.blob, ref_rp))
        same(run_eligible_ranked(case.topo, case.blob, rp, full, cls, 3), run_lw_ranked(case.topo, case.blob, ref_rp, 3))


@pytest.mark.parametrize("seed,n,k", [(1, 33, 2), (2, 130, 7), (4, 130, 64), (3, 33, 1)])
def test_placements_and_alternates_stay_on_admitted_nodes(seed, n, k):
    case = gg.make_case(seed, n, scarce=seed % 2 == 0, exclusive=True)
    topo, gblob = case.topo, case.blob
    rp = mixed_pods(gblob)
    cls = random_classes(n, k, seed)
    masks = random_masks(gblob, k, seed)
    a, s, d, sc, an, asc = run_eligible_ranked(topo, gblob, rp, masks, cls, 4)
    assert [x.tobytes() for x in (a, s, d)] == [x.tobytes() for x in run_eligible(topo, gblob, rp, masks, cls)]
    r0, checked = 0, 0
    for g, X in enumerate(groups_of(gblob, rp)):
        for ri in range(X.q):
            ok = admits(masks[r0 + ri], cls)
            first = X.pod0 + X.first_pod[ri]
            pods = np.arange(first, first + X.pending[ri] * X.S[ri])
            placed = a[pods][a[pods] >= 0]
            assert ok[placed].all() and np.isfinite(sc[pods][a[pods] >= 0]).all()
            alts = an[pods][an[pods] >= 0]
            assert ok[alts].all()
            checked += len(placed) + len(alts)
        r0 += X.q
    assert checked > 0


def test_placed_scores_equal_the_unmasked_rows():
    """A mask changes which entries are finite, never their value: with one anchor and one role, each placed pod's
    score is the unmasked oracle's row entry at its node."""
    n = 64
    topo = synth.make_topology(n, seed=5, tiers=2, max_free=4)
    topo.domain_owner = np.full(int(topo.domain.max()) + 1, -1, np.int32)
    cls = (np.arange(n) % 3).astype(np.int32)
    blob = build([Group(gid=1, roles=[(0, 3, 1, 0)], pair=[[1]], anchors=[(7, 0, 1)])])
    rp = [(1, -1)]
    a, s, d, sc, an, asc = run_eligible_ranked(topo, blob, rp, [0b101], cls, 2)
    rows = run_lw_rows(topo, blob, rp)[3]
    assert (a >= 0).all() and (cls[a] != 1).all()
    assert sc[0] == rows[(0, 0, 0)][a[0]]   # the first wave's row: no pod of the group placed yet


# ---- hand-built cases: name -> () -> dict(topo, blob, rp, masks, cls, n_alt, level_domain, expect(outputs))

def _flat(n, free=1):
    topo = synth.make_topology(n, seed=11, tiers=2, max_free=2)
    topo.domain_owner = np.full(int(topo.domain.max()) + 1, -1, np.int32)
    topo.free[:] = free
    return topo


def _best_node_excluded():
    n = 32
    topo = _flat(n, free=2)
    cls = np.zeros(n, np.int32)
    blob = build([Group(gid=1, roles=[(0, 1, 1, 0)], pair=[[1]])])
    best = int(lw.run_lw(topo, blob, [(1, -1)])[0][0])
    cls[best] = 1

    def expect(out):
        assert out[0][0] >= 0 and out[0][0] != best
    return dict(topo=topo, blob=blob, rp=[(1, -1)], masks=[0b01], cls=cls, n_alt=2, expect=expect)


def _dstar_moves():
    """The first participating role's best node is excluded: D* follows its best admitted node."""
    n = 32
    topo = _flat(n, free=2)
    topo.domain = (np.arange(n) // 8).astype(np.int32)
    topo.domain_owner = np.full(4, -1, np.int32)
    blob = build([Group(gid=1, roles=[(0, 1, 1, ROLE_EXCLUSIVE), (0, 1, 1, ROLE_EXCLUSIVE)], pair=[[1, 1], [1, 1]],
                        flags=STEP_EXCLUSIVE)])
    _, _, d0 = lw.run_lw(topo, blob, [(1, -1), (1, -1)])
    cls = (topo.domain == d0[0]).astype(np.int32)   # the whole unmasked D* is class 1

    def expect(out):
        a, s, d = out[:3]
        assert d[0] >= 0 and d[0] != d0[0] and (topo.domain[a] == d[0]).all()
    return dict(topo=topo, blob=blob, rp=[(1, -1), (1, -1)], masks=[0b01, ALL], cls=cls, n_alt=1, expect=expect)


def _coloc_domain_too_few_admitted():
    """A replica of 3 pods co-located at level 0: the best domain has only 2 admitted nodes, so it loses."""
    n = 32
    topo = _flat(n)
    topo.domain = (np.arange(n) // 4).astype(np.int32)
    topo.domain_owner = np.full(8, -1, np.int32)
    blob = build([Group(gid=1, roles=[(0, 1, 1, 0)], pair=[[1]])])
    a0 = lw.run_lw(topo, blob, [(3, 0)])[0]
    d_best = int(topo.domain[a0[0]])
    cls = np.zeros(n, np.int32)
    cls[np.flatnonzero(topo.domain == d_best)[:2]] = 1

    def expect(out):
        a = out[0]
        assert (a >= 0).all() and len(set(topo.domain[a].tolist())) == 1 and topo.domain[a[0]] != d_best
    return dict(topo=topo, blob=blob, rp=[(3, 0)], masks=[0b01], cls=cls, n_alt=2, expect=expect)


def _gang_fails():
    n = 16
    topo = _flat(n)
    cls = np.zeros(n, np.int32)
    cls[:3] = 1   # the role admits 3 nodes of free 1, it needs 4 pods
    blob = build([Group(gid=1, roles=[(0, 4, 1, 0)], pair=[[1]], flags=STEP_GANG)])

    def expect(out):
        a, s = out[:2]
        assert s[0] == 2 and (a == -1).all()
    return dict(topo=topo, blob=blob, rp=[(1, -1)], masks=[0b10], cls=cls, n_alt=3, expect=expect)


def _mask_zero():
    n = 16
    topo = _flat(n)
    blob = build([Group(gid=1, roles=[(0, 2, 1, 0), (0, 1, 1, 0)], pair=[[1, 0], [0, 1]])])

    def expect(out):
        a, s = out[:2]
        assert (a[:2] == -1).all() and a[2] >= 0 and s[0] == 1
    return dict(topo=topo, blob=blob, rp=[(1, -1), (1, -1)], masks=[0, ALL], cls=np.zeros(n, np.int32), n_alt=2,
                expect=expect)


def _anchor_on_excluded_node():
    """A scheduled pod on node m, which its role no longer admits, still lifts m's neighbours: the pod lands next to
    it, not where it would land without the anchor."""
    n = 64
    topo = synth.make_topology(n, seed=3, tiers=2, max_free=2)
    topo.domain_owner = np.full(int(topo.domain.max()) + 1, -1, np.int32)
    topo.free[:] = 1
    free_pick = int(lw.run_lw(topo, build([Group(gid=1, roles=[(0, 1, 1, 0)], pair=[[1]])]), [(1, -1)])[0][0])
    m = (free_pick + n // 2) % n
    cls = np.zeros(n, np.int32)
    cls[m] = 1
    blob = build([Group(gid=1, roles=[(0, 1, 1, 0)], pair=[[1]], anchors=[(m, 0, 1)])])
    nbrs = set(topo.col_idx[topo.row_ptr[m]:topo.row_ptr[m + 1]].tolist())

    def expect(out):
        a = out[0]
        assert a[0] != m and a[0] in nbrs and a[0] != free_pick
    return dict(topo=topo, blob=blob, rp=[(1, -1)], masks=[0b01], cls=cls, n_alt=2, expect=expect)


HAND_CASES = {
    "best_node_excluded": _best_node_excluded,
    "dstar_moves": _dstar_moves,
    "coloc_domain_too_few_admitted": _coloc_domain_too_few_admitted,
    "gang_fails": _gang_fails,
    "mask_zero": _mask_zero,
    "anchor_on_excluded_node": _anchor_on_excluded_node,
}


@pytest.mark.parametrize("name", sorted(HAND_CASES))
def test_hand_built_known_answers(name):
    c = HAND_CASES[name]()
    out = run_eligible_ranked(c["topo"], c["blob"], c["rp"], c["masks"], c["cls"], c["n_alt"])
    c["expect"](out)
    unmasked = run_lw_ranked(c["topo"], c["blob"], c["rp"], c["n_alt"])
    assert any(x.tobytes() != y.tobytes() for x, y in zip(out[:3], unmasked[:3]))   # the mask made the difference
