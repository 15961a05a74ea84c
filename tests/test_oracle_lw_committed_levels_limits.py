"""CPU: the preconditions of tests/lw_commit_levels_limits_cases.py asserted on the oracle of committed leader-worker
batches at levels (tests/lw_committed_levels_oracle.py) and its round replay: each case needs the term it was built
around, the churn and final-list facts hold round by round, the chains replay to exactly G rounds, the invariants hold
on the oracle's outputs, every ranked alternate breaks no anti-affinity term, and the coverage list names every
bullet."""
import numpy as np
import pytest

import levels_oracle as lo
import lw_commit_levels_gen as lvg
import lw_commit_levels_limits_cases as lc
from commit_levels_gen import KEYS
from lw_committed_oracle import groups_of
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE

CASES = lc.cases()
IDS = [c.name for c in CASES]


def invariants(c, a, s, d):
    """Capacity over the batch, whole replicas inside one level-C domain, the reference's anti-affinity terms, one gid
    per reported (level, domain) unless one of them was fixed to it."""
    gb, rp = c.blob(), c.role_pods()
    used = np.zeros(c.topo.n, np.int64)
    rep = {}
    for g, X in enumerate(groups_of(gb, rp)):
        for ri in range(X.q):
            lo_ = X.pod0 + X.first_pod[ri]
            pods = a[lo_:lo_ + X.pending[ri] * X.S[ri]].reshape(-1, X.S[ri])
            assert ((pods >= 0).all(axis=1) | (pods < 0).all(axis=1)).all(), (c.name, g, ri)
            for row in pods[pods[:, 0] >= 0]:
                if X.C[ri] >= 0:
                    assert len(set(c.lv[X.C[ri]][row].tolist())) == 1, (c.name, g, ri, row)
                np.add.at(used, row, X.demand[ri])
        grp = c.groups[g]
        if grp.flags & STEP_EXCLUSIVE and d[g] >= 0 and s[g] != 2:
            rep.setdefault((grp.level, int(d[g])), []).append((grp.gid, grp.fixed_domain >= 0))
    assert (used <= c.topo.free).all(), (c.name, np.nonzero(used > c.topo.free)[0][:8])
    for k, v in rep.items():
        if len({gid for gid, _ in v}) > 1:
            assert any(fx for _, fx in v), (c.name, k, v)
    assert lvg.violations(c.lv, c.occ, gb, rp, a, s) == [], c.name


@pytest.mark.parametrize("i", range(len(CASES)), ids=IDS)
def test_invariants_and_the_replay_end_on_the_oracle(i):
    c = CASES[i]
    a, s, d = c.expected()
    invariants(c, a, s, d)
    rs = lc.replay(c)
    assert lc.key(rs[-1]) == (a.tolist(), s.tolist(), d.tolist()), c.name
    assert 1 <= len(rs) <= len(c.groups)
    if c.rounds is not None:
        assert len(rs) == c.rounds, (c.name, len(rs))


@pytest.mark.parametrize("kind", ["pods", "shrink", "domain"])
def test_list_churn(kind):
    c = lc.churn(kind)
    f = lc.churn_facts(c)
    assert f["rounds"] == 3 and f["reader_moves"] and f["reader_in_zone"] and f["stale_differs"], f
    assert (f["before"], f["after"]) == {"pods": (2, 0), "shrink": (3, 1), "domain": (1, 0)}[kind], f


def test_claims_only_the_final_lists_carry():
    f = lc.final_lists_facts(lc.final_lists())
    assert f["rounds"] == 2 and f["last_changed"] and f["alt_differs"] and f["node1_removed"] and f["a_zone"] == 0, f


@pytest.mark.parametrize("G,kind", lc.CHAINS, ids=[f"{k}{G}" for G, k in lc.CHAINS])
def test_chains_take_exactly_G_rounds_through_their_term(G, kind):
    c = lc.chain(G, kind)
    f = lc.chain_facts(c)
    assert f["alternates"] and f["all_placed"] and f["replay_final"], f
    assert f["rounds"] == G == c.rounds, f
    if kind == "P":
        assert f["without_P"] and not f["without_K"], f
    elif kind == "K":
        assert f["without_K"] and not f["without_P"] and f["lmask"] == (1 << 3 | 1 << 6), f
    else:
        assert f["without_K"] and f["lmask"] == 0xFF, f


def test_refresh_chain_replays_to_exactly_its_length():
    c = lc.chain(*lc.REFRESH_CHAIN)
    f = lc.chain_facts(c)
    assert f["alternates"] and f["all_placed"] and f["lmask"] == 0xFF and f["replay_final"], f
    assert f["rounds"] == lc.REFRESH_CHAIN[0] == c.rounds, f


@pytest.mark.parametrize("i", range(4))
def test_all_eight_levels_and_sparse_masks(i):
    c = lc.levels_cases()[i]
    f = lc.levels_facts(c)
    ex, ot = c.extra["excl"], c.extra["other"]
    assert f["lmask"] == sum(1 << L for L in ex) and f["excl"] == set(ex) and f["other"] == set(ot), f
    assert set(c.extra["pairs"]) <= f["pairs"] and f["placed"] > 0 and f["multi_pod"], f
    assert f["without_K"] or f["without_P"], f
    if "specs" in c.extra:                    # the sparse masks: every claim moves its reader, through K and P
        m = lc.moved_facts(c)
        assert all(m["moved"]) and all(m["held"]) and f["without_K"] and f["without_P"], (f, m)


@pytest.mark.parametrize("kind", ["report", "pods", "idle"])
def test_level_offset_edges(kind):
    c = lc.offsets(kind)
    f = lc.offsets_facts(c)
    assert f["claimed_all"] and f["levels"] == 8 and f["idle"] == (14 if kind == "idle" else 0), f
    assert len(f["moved"]) == 14 and all(f["moved"]), f


@pytest.mark.parametrize("kind", ["edge", "random"])
def test_long_pod_lists(kind):
    f = lc.long_pods_facts(lc.long_pods(kind))
    assert f["pods_in_zone0"] >= 2048 and f["readers"][0] == 1 and f["without_P"], f
    assert f["nests"] == (kind == "edge"), f


def test_opted_out_roles_stay_out_of_p():
    f = lc.opted_out_facts(lc.opted_out())
    assert f["opted_out"] == [1] * 4 and f["reader"] == [1, 1] and f["participating"] == [12, 12], f
    assert f["counted_differs"], f


def test_gang_failure_mid_chain_drops_every_claim():
    f = lc.gang_mid_chain_facts(lc.gang_mid_chain())
    assert f["rounds"] == 3 and f["f_round1"] == 0 and f["f_final"] == 2 and f["f_claims_final"], f
    assert f["reader"] == [3, 8, 3] and f["kept_report_differs"], f


def test_gids():
    f = lc.gids_facts(lc.gids())
    assert f["gid_ends"] and f["shared_gid_matters"] and f["first_differs"], f
    assert f["own_pods_zone"] == f["first77_zone"] and f["reporters"] == [5, 5] and f["last_keeps_out"] == -1, f


def test_mixed_level_emit_blocks():
    f = lc.emit_blocks_facts(lc.emit_blocks())
    assert f["steps"] >= 33 and f["one_wave"] and f["adjacent_mixed"] >= 32 and 0 < f["non_exclusive"] < 10, f
    assert f["without_K"] and f["without_P"], f


@pytest.mark.parametrize("n", [4097, 129])
def test_ragged_chunks(n):
    f = lc.ragged_facts(lc.ragged(n))
    assert f["first_last"] == n - 1 and all(f["straddle"]) and f["placed"] >= 2, f


def alternate_breaks_a_term(c, gb, rp, a, s, p, m) -> bool:
    """Does pod p moved to node m break an anti-affinity term?  Only pairs with p change, so p's labelled pod is
    checked against the records and every other placed participating pod (levels_oracle.violates: both directions)."""
    levels = [g.level for g in c.groups]
    others, me = [tuple(int(x) for x in r) for r in np.asarray(c.occ).reshape(-1, 3)], None
    for g, X in enumerate(groups_of(gb, rp)):
        if not X.flags & STEP_EXCLUSIVE or s[g] == 2:
            continue
        for ri in range(X.q):
            if not X.rflags[ri] & ROLE_EXCLUSIVE:
                continue
            lo_ = X.pod0 + X.first_pod[ri]
            for q in range(lo_, lo_ + X.pending[ri] * X.S[ri]):
                if q == p:
                    me = (X.gid, levels[g])
                elif a[q] >= 0:
                    others.append((int(a[q]), X.gid, levels[g]))
    if me is None:
        return False
    return lo.violates(c.lv, KEYS[:len(c.lv)], np.array(others, np.int64).reshape(-1, 3), me[0], me[1], int(m))


@pytest.mark.parametrize("i", range(len(CASES)), ids=IDS)
def test_ranked_alternates_break_no_term(i):
    c = CASES[i]
    gb, rp = c.blob(), c.role_pods()
    a, s, d, score, alt, _ = c.expected_ranked(4)
    assert np.array_equal(a, c.expected()[0])
    for g, X in enumerate(groups_of(gb, rp)):
        for ri in range(X.q):
            lo_ = X.pod0 + X.first_pod[ri]
            for p in range(lo_, lo_ + X.pending[ri] * X.S[ri]):
                for m in alt[p][alt[p] >= 0]:
                    assert not alternate_breaks_a_term(c, gb, rp, a, s, p, m), (c.name, g, p, m)
                    if X.C[ri] >= 0:
                        assert c.lv[X.C[ri]][m] == c.lv[X.C[ri]][a[p]]


def test_coverage():
    cov = lc.coverage(CASES)
    cov.update(lc.scale_and_bound_coverage())
    assert set(cov) == set(lc.BULLETS) and all(cov.values()), [k for k, v in cov.items() if not v]
