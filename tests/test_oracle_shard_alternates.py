"""CPU: a numpy model of ranked alternates on node-axis shards (DESIGN.md §3.17), against the world = 1 oracles.

Each rank keeps, per ranked row, the ALT_LIST (= 9) best candidates of its slab by key (score descending, node
ascending), its own node included; the merge takes the best 9 of the world lists, rank-major, drops the replica's
own node and keeps n_alt.  The slabs are those of the library: rank g starts at g * n / world rounded down to 128, so
some slabs are empty at small n.  The model must give alternates_oracle's and committed_alternates_oracle's outputs
on generated fleets at world 1, 2, 3, 4 and 8, and the plain sort on hand-made rows: the best nodes all in one slab,
the replica's own node as the global best in another rank's slab, equal scores on both sides of a slab bound."""
import numpy as np
import pytest

import commit_gen as cg
import committed_alternates_oracle as cao
import committed_oracle as co
import groups_gen as gg
from alternates_oracle import _key, run_fleet_ranked
from oracle import wave_loop

ALT_LIST = 9
WORLDS = [1, 2, 3, 4, 8]


def slab_bounds(n, world):
    return [0 if g == 0 else n if g == world else g * n // world // 128 * 128 for g in range(world + 1)]


def best(S, idx, k):
    """The k best of nodes idx by key: score descending, node ascending."""
    idx = np.asarray(idx, dtype=np.int64)
    return idx[np.lexsort((idx, -S[idx].astype(np.float64)))][:k]


def shard_rank(S, ok, own, n_alt, bounds):
    """The protocol: per-slab top ALT_LIST lists (own node included), the rank-major merge, own node dropped."""
    lists = [best(S, lo + np.nonzero(ok[lo:hi])[0], ALT_LIST) for lo, hi in zip(bounds, bounds[1:])]
    merged = best(S, np.concatenate(lists), ALT_LIST)
    return [int(m) for m in merged if m != own][:n_alt]


def plain_rank(S, ok, own, n_alt):
    ok = ok.copy()
    ok[own] = False
    return [int(m) for m in best(S, np.nonzero(ok)[0], n_alt)]


def ranked_rows(topo, groups, rows_of, ok_of, n_alt, bounds):
    """(score, alt_node, alt_score) through the model, in assign order; rows_of / ok_of as the oracles build them."""
    score, alt_node, alt_score = [], [], []
    for s, res, k, role, node in rows_of():
        if node < 0:
            score.append(-np.inf)
            alt_node.append([-1] * n_alt)
            alt_score.append([-np.inf] * n_alt)
            continue
        S = k
        alts = shard_rank(S, ok_of(s, res, role, S), node, n_alt, bounds)
        score.append(float(S[node]))
        alt_node.append(alts + [-1] * (n_alt - len(alts)))
        alt_score.append([float(S[x]) for x in alts] + [-np.inf] * (n_alt - len(alts)))
    R = len(score)
    return (np.asarray(score, np.float32), np.asarray(alt_node, np.int32).reshape(R, n_alt),
            np.asarray(alt_score, np.float32).reshape(R, n_alt))


def model_plain(topo, groups, n_alt, world):
    """alternates_oracle.run_fleet_ranked's rows and candidate rule (own node kept), ranked through the model."""
    rows = {}

    def on_wave(w, active, blob, r):
        off = 0
        for s in active:
            for ri, ordinal, cnt in s.waves[w]:
                row = np.array(r["matrix"][off], dtype=np.float32, copy=True)
                for c in range(cnt):
                    rows[_key(s.g, ri, ordinal + c)] = row
                off += cnt

    states, _ = wave_loop.run_fleet(topo, groups, want_matrix=True, on_wave=on_wave)
    free = np.asarray(topo.free, np.int64)
    domain = np.asarray(topo.domain, np.int64)
    used = {}
    for s in states:
        res = s.result()
        u = np.zeros(len(free), np.int64)
        for ri in s.order:
            for c in range(s.pending[ri]):
                node = res["nodes"][_key(s.g, ri, s.first[ri] + c)]
                if node >= 0:
                    u[node] += s.g.roles[ri].demand
        used[id(s)] = u

    def rows_of():
        for s in states:
            res = s.result()
            for ri in s.order:
                for c in range(s.pending[ri]):
                    k = _key(s.g, ri, s.first[ri] + c)
                    node = res["nodes"][k]
                    yield s, res, rows.get(k), s.g.roles[ri], node

    def ok_of(s, res, role, S):
        ok = (S != -np.inf) & (free - used[id(s)] >= role.demand)
        if s.g.exclusive and role.exclusive:
            ok &= domain == res["domain"]
        return ok

    return ranked_rows(topo, groups, rows_of, ok_of, n_alt, slab_bounds(len(free), world))


def model_committed(topo, groups, n_alt, world):
    """committed_alternates_oracle's rows and candidate rule at level 0 (own node kept), ranked through the model."""
    states, rows = cao.run_committed_rows(topo, groups, fast=True)
    free = np.asarray(topo.free, np.int64)
    used = np.zeros(len(free), np.int64)
    for s in states:
        for node, amt in co.group_claims(s).items():
            used[node] += amt
    dom = np.asarray(topo.domain, np.int64)
    last = np.full(len(topo.domain_owner), cao.FREE, np.int32)
    for s in states:
        res = s.result()
        if s.g.exclusive and res["status"] != 2 and res["domain"] >= 0:
            last[res["domain"]] = s.g.gid
    owner = np.array(topo.domain_owner, dtype=np.int32, copy=True)
    owner[last != cao.FREE] = last[last != cao.FREE]
    owner = owner[dom]

    def rows_of():
        for s in states:
            res = s.result()
            for ri in s.order:
                for c in range(s.pending[ri]):
                    k = cao._key(s.g, ri, s.first[ri] + c)
                    yield s, res, rows.get(k), s.g.roles[ri], res["nodes"][k]

    def ok_of(s, res, role, S):
        ok = (S != -np.inf) & (free - used >= role.demand)
        if s.g.exclusive and role.exclusive:
            ok &= (dom == res["domain"]) & ((owner == cao.FREE) | (owner == s.g.gid))
        return ok

    return ranked_rows(topo, groups, rows_of, ok_of, n_alt, slab_bounds(len(free), world))


def bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


def same(got, exp):
    sc, an, asc = got
    assert np.array_equal(bits(sc), bits(exp[3]))
    assert np.array_equal(an, exp[4]) and np.array_equal(bits(asc), bits(exp[5]))


@pytest.mark.parametrize("seed,n,scarce,excl", gg.CASES)
def test_model_equals_alternates_oracle(seed, n, scarce, excl):
    case = gg.make_case(seed, n, scarce=scarce, exclusive=excl)
    groups = wave_loop.groups_from_blob(case.blob)
    exp = run_fleet_ranked(case.topo, groups, 8)
    for world in WORLDS:
        same(model_plain(case.topo, groups, 8, world), exp)


@pytest.mark.parametrize("i", range(0, len(cg.cases()), 2))
def test_model_equals_committed_alternates_oracle(i):
    case = cg.cases()[i]
    groups = wave_loop.groups_from_blob(case.blob)
    exp = cao.run_fleet_committed_ranked(case.topo, groups, 8, fast=True)
    for world in WORLDS:
        same(model_committed(case.topo, groups, 8, world), exp)


def test_slab_bounds_leave_empty_slabs_at_small_n():
    assert slab_bounds(300, 4) == [0, 0, 128, 128, 300]
    assert slab_bounds(4097, 8) == [0, 512, 1024, 1536, 2048, 2560, 3072, 3584, 4097]


@pytest.mark.parametrize("world", WORLDS)
def test_hand_made_rows(world):
    n = 1100
    bounds = slab_bounds(n, world)
    rng = np.random.default_rng(world)
    cases = []
    # the best nodes of the row all in one slab (the last one)
    S = rng.uniform(0, 1, n).astype(np.float32)
    S[bounds[-2]:bounds[-2] + 12] += 2
    cases.append((S, np.ones(n, bool), 5))
    # the replica's own node is the global best and lies in another rank's slab than the next best
    S = rng.uniform(0, 1, n).astype(np.float32)
    S[n - 3] = 5.0
    S[:10] += 1
    cases.append((S, np.ones(n, bool), n - 3))
    # equal scores on both sides of every slab bound: node ascending decides
    S = np.full(n, 0.5, np.float32)
    for b in bounds[1:-1]:
        S[max(0, b - 6):b + 6] = 1.0
    cases.append((S, np.ones(n, bool), 0))
    # few candidates (fewer than n_alt), -inf elsewhere
    S = np.full(n, -np.inf, np.float32)
    S[[3, 700, 1099]] = [1.0, 2.0, 1.0]
    cases.append((S, S != -np.inf, 700))
    for S, ok, own in cases:
        for n_alt in (0, 1, 8):
            assert shard_rank(S, ok, own, n_alt, bounds) == plain_rank(S, ok, own, n_alt), (world, own, n_alt)
