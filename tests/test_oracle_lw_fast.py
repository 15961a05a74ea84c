"""CPU: the one-pass choice of a replica's co-location domain (lw_oracle.domain_fast) against the literal enumeration of
rule 3 (lw_oracle.domain_literal), wave for wave: every place_wave call of run_lw and run_lw_committed is made with
both and must give the same (pods, status, D*).  Generated fleets of tests/groups_gen.py and tests/lw_commit_gen.py
with co-location at level 0, one domain per node, racks of 16 and one domain for the whole fleet; demand 0, S = 32 and
scarce capacity."""
import numpy as np
import pytest

import groups_gen as gg
import lw_commit_gen as lg
import lw_oracle as lw
from lw_alternates_oracle import run_lw_ranked
from lw_committed_oracle import run_lw_committed


def levels(topo):
    n = topo.n
    return [topo.domain, np.arange(n, dtype=np.int32), (np.arange(n) // 16).astype(np.int32), np.zeros(n, np.int32)]


class Both:
    """Stands in for lw.place_wave: runs the literal and the fast form on the same inputs, asserts they agree."""

    def __init__(self):
        self.calls = self.coloc = 0

    def __call__(self, G, w, rows, topo, excl_domain, level_domain):
        a = lw._place_wave(G, w, rows, topo, excl_domain, level_domain)
        b = lw._place_wave(G, w, rows, topo, excl_domain, level_domain, choose=lw.domain_fast)
        assert a[0] == b[0] and a[1:] == b[1:], (G.gid, w, a, b)
        self.calls += 1
        self.coloc += any(G.C[ri] >= 0 for ri, _, _ in G.waves[w])
        return a


@pytest.fixture
def both(monkeypatch):
    b = Both()
    monkeypatch.setattr(lw, "place_wave", b)
    return b


def cycle(gblob, S, C):
    k = iter(range(1 << 20))
    return lw.role_pods_for(gblob, lambda g, r: (S[(g + r) % len(S)], C[next(k) % len(C)]))


@pytest.mark.parametrize("seed,n,scarce,excl", [c for c in gg.CASES if c[1] <= 130])
@pytest.mark.parametrize("S", [(2, 4, 1), (3, 1), (4, 2)])
def test_generated_fleets_wave_for_wave(both, seed, n, scarce, excl, S):
    """(S = 32 on these fleets would leave the exactness bound: the committed fleets below and the random rows carry it.)"""
    case = gg.make_case(seed, n, scarce=scarce, exclusive=excl)
    lw.run_lw(case.topo, case.blob, cycle(case.blob, S, (0, 1, 2, 3, -1)), level_domain=levels(case.topo))
    assert both.coloc > 0


@pytest.mark.parametrize("seed,n,scarce", lg.SEEDS)
def test_committed_fleets_wave_for_wave(both, seed, n, scarce):
    f = lg.fleet(seed, n, n_groups=14, scarce=scarce, levels=True, S_max=32)
    lv = list(f.lv) + [np.zeros(n, np.int32)]
    rp = f.role_pods().copy()
    rp[::3, 1] = 3                                   # one domain for the whole fleet
    run_lw_committed(f.topo, f.blob(), rp, level_domain=lv)
    assert both.calls > 0


def test_fast_domains_swaps_every_oracle():
    """Inside fast_domains() the three oracles give what they give with the literal form; outside, place_wave is the
    literal one again."""
    case = gg.make_case(4, 130, scarce=True, exclusive=True)
    lv = levels(case.topo)
    rp = cycle(case.blob, (4, 3, 2), (1, 2, 0, 3))
    slow = (lw.run_lw(case.topo, case.blob, rp, level_domain=lv),
            run_lw_ranked(case.topo, case.blob, rp, 8, level_domain=lv),
            run_lw_committed(case.topo, case.blob, rp, level_domain=lv))
    with lw.fast_domains():
        assert lw.place_wave is not lw._place_wave
        fast = (lw.run_lw(case.topo, case.blob, rp, level_domain=lv),
                run_lw_ranked(case.topo, case.blob, rp, 8, level_domain=lv),
                run_lw_committed(case.topo, case.blob, rp, level_domain=lv))
    assert lw.place_wave is lw._place_wave
    for x, y in zip(slow, fast):
        for u, v in zip(x, y):
            assert np.array_equal(np.asarray(u).view(np.uint8), np.asarray(v).view(np.uint8))
    assert (slow[0][0] >= 0).any() and (slow[0][0] < 0).any()


@pytest.mark.parametrize("seed", range(40))
def test_domain_choice_on_random_rows(seed):
    """The two forms of D_r on random candidates: ties in score, demand 0 and 1 .. 3, S up to 32, free near the
    cut-offs floor(room / demand) = S - 1, S, S + 1, partitions from one domain per node to one domain."""
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 300))
    row = rng.integers(0, 4, size=n).astype(np.float32)
    row[rng.random(n) < 0.2] = -np.inf
    S = int(rng.choice([1, 2, 3, 31, 32]))
    demand = int(rng.choice([0, 1, 2, 3]))
    avail = rng.integers(0, 3, size=n).astype(np.int64)
    if demand:
        avail[rng.random(n) < 0.1] = rng.choice([S - 1, S, S + 1]) * demand
    dom = (np.arange(n) // int(rng.choice([1, 4, 16, n]))).astype(np.int32)
    if rng.random() < 0.5:
        dom = rng.permutation(dom)
    cand = (row != -np.inf) & (avail >= demand)
    assert lw.domain_fast(cand, avail, demand, S, dom, row) == lw.domain_literal(cand, avail, demand, S, dom, row)
