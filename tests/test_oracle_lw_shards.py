"""CPU: numpy models of leader-worker placement on node-axis shards (DESIGN.md §3.18), against the world = 1 oracles.

1. The replicated evaluator.  Every rank evaluates a row entry from the snapshot instead of reading the dense row:
     v_p(n) = -inf  if free[n] < demand_p, (participating row of an exclusive step) owner(n) not in {-1, gid}, or
                    free[n] - consumed[n] < demand_p;
            = need_p·base[n] + sum over anchors (m, q, c) with n in N[m] ∪ {m} of pair[p][q]·c·w(n, m)
              (self weight RBGTOPO_SELF_W·c), base[n] = sum_j w_j·min(free[col_j], F) + SELF_W·min(free[n], F).
   It must equal, bit for bit over all nodes, every dense row the oracle (oracle/placer.py) scores for the leader-worker
   oracles: consumed records, anchors, exclusive owners, the level-0 claims of committed batches (the oracles hand them
   over as domain owners) and committed batches at levels (level views).
2. The pod-job exchange.  Per ranked job, each rank keeps the ALT_LIST (= 9) best candidates of its slab (the pod's
   own node included, inside the replica's co-location domain); the merge takes the best 9 of the world lists, drops
   the pod's own node and keeps n_alt.  Run inside the ranked leader-worker oracles at world 1, 2, 3, 4 and 8 with
   the library's slab bounds, it must give their outputs unchanged."""
import numpy as np
import pytest

import groups_gen as gg
import lw_alternates_oracle as lwa
import lw_commit_gen as lg
import lw_commit_levels_gen as lvg
import lw_committed_alternates_oracle as lcao
import lw_oracle as lw
from oracle import placer as oracle_placer
from test_oracle_shard_alternates import ALT_LIST, WORLDS, shard_rank, slab_bounds

HDR, SW = 8, 16
F_CAP, SELF_W = 8, 8000


def base_of(topo):
    rp, col, w = (np.asarray(a, np.int64) for a in (topo.row_ptr, topo.col_idx, topo.edge_w))
    fmin = np.minimum(np.asarray(topo.free, np.int64), F_CAP)
    rows = np.repeat(np.arange(len(fmin)), np.diff(rp))
    base = np.zeros(len(fmin), np.int64)
    np.add.at(base, rows, w * fmin[col])
    return base + SELF_W * fmin


def model_rows(topo, blob):
    """The dense rows of a step blob through v_p(n), one per role row of every step: [(step, p, count, row)]."""
    blob = np.asarray(blob, np.int64)
    rp, col, w = (np.asarray(a, np.int64) for a in (topo.row_ptr, topo.col_idx, topo.edge_w))
    free = np.asarray(topo.free, np.int64)
    n = len(free)
    base = base_of(topo)
    owner = np.asarray(topo.domain_owner, np.int64)[np.asarray(topo.domain, np.int64)]
    out = []
    for s in range(int(blob[2])):
        st = blob[HDR + SW * s:HDR + SW * (s + 1)]
        gid, flags, P, Q, na, nc = int(st[0]), int(st[1]), int(st[3]), int(st[5]), int(st[7]), int(st[9])
        roles = blob[st[4]:st[4] + 4 * P].reshape(P, 4)
        pair = blob[st[6]:st[6] + P * Q].reshape(P, Q)
        delta = np.zeros((P, n), np.int64)
        for m, q, c in blob[st[8]:st[8] + 3 * na].reshape(na, 3):
            nb = col[rp[m]:rp[m + 1]]
            delta[:, nb] += pair[:, q, None] * c * w[rp[m]:rp[m + 1]][None, :]
            delta[:, m] += pair[:, q] * SELF_W * c
        consumed = np.zeros(n, np.int64)
        con = blob[st[10]:st[10] + 2 * nc].reshape(nc, 2)
        np.add.at(consumed, con[:, 0], con[:, 1])
        for p in range(P):
            count, demand, need, rflags = (int(x) for x in roles[p])
            bad = (free < demand) | (free - consumed < demand)
            if (flags & lw.STEP_EXCLUSIVE) and (rflags & lw.ROLE_EXCLUSIVE):
                bad |= ~((owner == -1) | (owner == gid))
            v = (need * base + delta[p]).astype(np.float32)
            v[bad] = -np.inf
            out.append((s, p, count, v))
    return out


@pytest.fixture
def evaluator_checked(monkeypatch):
    """Every oracle scoring of the test checked against model_rows; yields the count of rows compared."""
    inner = oracle_placer.place
    seen = [0]

    def place(topo, blob, *a, **kw):
        r = inner(topo, blob, *a, **kw)
        if r["rc"] == 0 and r.get("matrix") is not None:
            row = 0
            for s, p, count, v in model_rows(topo, blob):
                got = np.asarray(r["matrix"][row], np.float32)
                assert np.array_equal(got.view(np.uint32), v.view(np.uint32)), \
                    (s, p, np.nonzero(got.view(np.uint32) != v.view(np.uint32))[0][:8])
                seen[0] += 1
                row += count
        return r
    monkeypatch.setattr(oracle_placer, "place", place)
    yield seen
    assert seen[0] > 0


def cycle_pods(gblob, S=(2, 4, 1), C=(-1, 0)):
    k = iter(range(1 << 20))
    return lw.role_pods_for(gblob, lambda g, r: (S[(g + r) % len(S)], C[next(k) % len(C)]))


@pytest.mark.parametrize("seed,n,scarce,excl", gg.CASES)
def test_evaluator_equals_the_rows_of_place_groups_lw(evaluator_checked, seed, n, scarce, excl):
    case = gg.make_case(seed, n, scarce=scarce, exclusive=excl)
    lw.run_lw(case.topo, case.blob, cycle_pods(case.blob))
    lw.run_lw(case.topo, case.blob, cycle_pods(case.blob, S=(4, 2), C=(0,)))


@pytest.mark.parametrize("seed,n,scarce", lg.SEEDS)
@pytest.mark.parametrize("mode", ["map", "occupancy"])
def test_evaluator_equals_the_rows_of_committed_batches(evaluator_checked, seed, n, scarce, mode):
    """Consumed records of earlier groups and the level-0 claims (map mode: the claim replaces the owner; occupancy:
    merged into owner_0)."""
    occ = mode == "occupancy"
    f = lg.fleet(seed, n, n_groups=14, scarce=scarce, levels=occ, occupancy=occ)
    kw = dict(level_domain=list(f.lv), owner0=lg.owner0(f)) if occ else {}
    lcao.run_lw_committed_rows(f.topo, f.blob(), f.role_pods(), **kw)


@pytest.mark.parametrize("seed,n,scarce,kind", lvg.SEEDS)
def test_evaluator_equals_the_rows_of_committed_batches_at_levels(evaluator_checked, seed, n, scarce, kind):
    f = lvg.fleet(seed, n, n_groups=14, scarce=scarce, kind=kind)
    f.expected()


def exchange(bounds):
    """lw_alternates_oracle.ranked_candidates through the pod-job exchange: the merged list (own node dropped)."""
    def candidates(row, node, free, used, demand, excl_mask, coloc_dom):
        ok = (row != -np.inf) & (free - used >= demand)   # the pod's own node stays in its slab's list
        if excl_mask is not None:
            ok &= excl_mask
        if coloc_dom is not None:
            ok &= coloc_dom == coloc_dom[node]
        out = np.zeros(len(row), bool)
        out[shard_rank(row, ok, node, ALT_LIST, bounds)] = True
        return out
    return candidates


def bits(x):
    x = np.asarray(x)
    return x.view(np.uint32) if x.dtype == np.float32 else x


def same(got, exp):
    for x, y in zip(got, exp):
        assert np.array_equal(bits(x), bits(y))


@pytest.mark.parametrize("seed,n,scarce,excl", gg.CASES)
def test_exchange_equals_lw_ranked(monkeypatch, seed, n, scarce, excl):
    case = gg.make_case(seed, n, scarce=scarce, exclusive=excl)
    rp = cycle_pods(case.blob)
    exp = lwa.run_lw_ranked(case.topo, case.blob, rp, 8)
    for world in WORLDS:
        monkeypatch.setattr(lwa, "ranked_candidates", exchange(slab_bounds(case.topo.n, world)))
        same(lwa.run_lw_ranked(case.topo, case.blob, rp, 8), exp)
        monkeypatch.undo()


@pytest.mark.parametrize("seed,n,scarce", lg.SEEDS)
@pytest.mark.parametrize("mode", ["map", "occupancy"])
def test_exchange_equals_lw_committed_ranked(monkeypatch, seed, n, scarce, mode):
    occ = mode == "occupancy"
    f = lg.fleet(seed, n, n_groups=14, scarce=scarce, levels=occ, occupancy=occ)
    kw = dict(level_domain=list(f.lv), owner0=lg.owner0(f)) if occ else {}
    exp = lcao.run_lw_committed_ranked(f.topo, f.blob(), f.role_pods(), 8, **kw)
    assert (exp[4] >= 0).any()
    for world in WORLDS:
        monkeypatch.setattr(lcao, "ranked_candidates", exchange(slab_bounds(f.topo.n, world)))
        same(lcao.run_lw_committed_ranked(f.topo, f.blob(), f.role_pods(), 8, **kw), exp)
        monkeypatch.undo()
