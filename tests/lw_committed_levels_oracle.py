"""Oracle of committed leader-worker batches at exclusive levels (rbgtopo_place_groups_lw_committed[_ranked] on a ctx
with RBGTOPO_CFG_LW_COMMIT_LEVELS, DESIGN.md §3.16; test infrastructure).  It composes existing pieces without
restating them:
  * group g runs lw_committed_oracle.run_group (the §3.11 loop, `consumed` seeded with every pod an earlier group
    placed) on levels_view.level_view of committed_levels_oracle.level_owner: owner_{L_g} ⊕ K ⊕ P, where K merges the
    gid of the last earlier exclusive reporter (status != 2) of dom_L(n) at every level L, and P the gid of every placed
    participating POD of an earlier exclusive group keyed at another level, in dom_{L_g}(n);
  * the ranked form keeps the row of every (group, wave, role) where run_group hands it to lw_oracle.place_wave and
    applies §3.15 with the owner after the whole batch counted at levels (own_B,g = level_owner over every group);
    co-location reads the caller's partitions."""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np

import levels_oracle
import levels_view
import lw_committed_oracle as lco
import lw_oracle as lw
from committed_levels_oracle import group_levels, level_owner
from lw_alternates_oracle import ranked_candidates

FREE = levels_oracle.FREE


def participating_pods(X: lw.LwGroup, assign: np.ndarray) -> List[int]:
    """Nodes of the placed pods of the group's participating (exclusive) roles."""
    out = []
    for ri in range(X.q):
        if X.rflags[ri] & lw.ROLE_EXCLUSIVE:
            lo = X.pod0 + X.first_pod[ri]
            out += [int(m) for m in assign[lo:lo + X.pending[ri] * X.S[ri]] if m >= 0]
    return out


def batch_claims(G: Sequence[lw.LwGroup], levels, status, domain, assign, n_domains, n_levels: int):
    """(last, pods) over the whole batch: last[L][d] = gid of the last exclusive reporter of d at L, pods = (gid, level,
    node) of every placed participating pod of an exclusive group; gang-failed groups claim nothing."""
    last = [np.full(int(n_domains[L]), FREE, np.int32) for L in range(n_levels)]
    pods = []
    for g, X in enumerate(G):
        if not (X.flags & lw.STEP_EXCLUSIVE) or status[g] == 2:
            continue
        if domain[g] >= 0:
            last[levels[g]][domain[g]] = X.gid
        pods += [(X.gid, levels[g], m) for m in participating_pods(X, assign)]
    return last, pods


def place_group(topo, dom, owner, n_domains, X: lw.LwGroup, L: int, claimed, last, pods, other: int,
                assign: np.ndarray):
    """Group X at exclusive level L against what the groups before it left: `claimed` (node -> demand), `last`
    (per level the gid of a domain's reporter) and `pods` ((gid, level, node) of their participating pods).  Writes its
    pods into `assign`; returns (status, domain)."""
    X.consumed = dict(claimed)
    ow = np.array(owner, dtype=np.int32, copy=True)
    ow[L] = level_owner(dom, owner, n_domains, L, last, pods)
    t = levels_view.level_view(topo, dom, ow, n_domains, L, X.gid, other)
    if X.fixed >= 0:    # the view numbers domain d of level L as 2d (2d + 1 for its nodes blocked to g)
        X.fixed *= 2
    lco.run_group(t, X, list(dom), t.domain, assign)
    if X.fixed >= 0:
        X.fixed //= 2
    if X.failed:
        assign[X.pod0:X.pod0 + X.n_pods] = -1
        return 2, -1
    return X.status, (X.fixed if X.flags & lw.STEP_EXCLUSIVE else -1)


def group_claims(X: lw.LwGroup, assign: np.ndarray, status: int, domain: int):
    """What a placed group takes from the groups after it: ({node: demand} of its placed pods, the domain it reports
    (-1 = none), the nodes of its placed participating pods); a gang-failed group takes nothing."""
    if status == 2:
        return {}, -1, []
    cap = {}
    for ri in range(X.q):
        lo = X.pod0 + X.first_pod[ri]
        for node in assign[lo:lo + X.pending[ri] * X.S[ri]]:
            if node >= 0:
                cap[int(node)] = cap.get(int(node), 0) + X.demand[ri]
    if not X.flags & lw.STEP_EXCLUSIVE:
        return cap, -1, []
    return cap, int(domain), participating_pods(X, assign)


def run_lw_committed_levels(topo, gblob, role_pods, level_domain, owner, n_domains, limit: Optional[int] = None,
                            terms: Sequence[str] = ("K", "P"), reporter: str = "last"):
    """(assign per pod, status[ng], domain[ng]).  level_domain [n_levels + 1][n] (row 0 = the snapshot's domain), owner
    = levels_oracle.derive_level_owner(level_domain, occ), n_domains per level; `limit`: place only the first `limit`
    groups (the rest keep -1 / -9 / -9).  `terms` / `reporter` exist for the tests' preconditions: the owner without
    K or P, or with the first earlier reporter of a domain instead of the last."""
    assert set(terms) <= {"K", "P"} and reporter in ("last", "first")
    dom = np.asarray(level_domain)
    G = lco.groups_of(gblob, role_pods)
    levels = group_levels(gblob)
    ng = len(G)
    assign = np.full(sum(X.n_pods for X in G), -1, dtype=np.int32)
    status = np.full(ng, -9, dtype=np.int32)
    domain = np.full(ng, -9, dtype=np.int32)
    last = [np.full(int(n_domains[L]), FREE, np.int32) for L in range(dom.shape[0])]
    pods: List = []
    claimed = {}
    other = levels_oracle.unused_gid({X.gid for X in G})
    for g in range(ng if limit is None else min(limit, ng)):
        X, L = G[g], levels[g]
        status[g], domain[g] = place_group(topo, dom, owner, n_domains, X, L, claimed, last, pods, other, assign)
        cap, rep, mine = group_claims(X, assign, status[g], domain[g])
        for node, amt in cap.items():
            claimed[node] = claimed.get(node, 0) + amt
        if rep >= 0 and "K" in terms and (reporter == "last" or last[L][rep] == FREE):
            last[L][rep] = X.gid
        if "P" in terms:
            pods += [(X.gid, L, m) for m in mine]
    return assign, status, domain


def run_lw_committed_levels_ranked(topo, gblob, role_pods, n_alt: int, level_domain, owner, n_domains, claims=None):
    """(assign, status, domain, score[P], alt_node[P, n_alt], alt_score[P, n_alt]) of §3.16's ranked form.  `claims`
    ((last, pods) as batch_claims gives them) replaces the batch's own claims in the ranking, for the tests'
    preconditions."""
    first_pod = {X.pod0: g for g, X in enumerate(lco.groups_of(gblob, role_pods)) if X.n_pods}
    rows = {}
    inner = lw.place_wave

    def keep(X, w, wave_rows, *args):
        for p, row in enumerate(wave_rows):
            rows[(first_pod[X.pod0], w, p)] = np.array(row, dtype=np.float32, copy=True)
        return inner(X, w, wave_rows, *args)

    lw.place_wave = keep
    try:
        assign, status, domain = run_lw_committed_levels(topo, gblob, role_pods, level_domain, owner, n_domains)
    finally:
        lw.place_wave = inner
    dom = np.asarray(level_domain)
    free = np.asarray(topo.free, dtype=np.int64)
    G = lco.groups_of(gblob, role_pods)
    levels = group_levels(gblob)
    used = np.zeros(len(free), dtype=np.int64)
    for g, X in enumerate(G):
        for ri in range(X.q):
            lo = X.pod0 + X.first_pod[ri]
            for node in assign[lo:lo + X.pending[ri] * X.S[ri]]:
                if node >= 0:
                    used[node] += X.demand[ri]
    last, pods = batch_claims(G, levels, status, domain, assign, n_domains, dom.shape[0]) if claims is None else claims
    P = len(assign)
    score = np.full(P, -np.inf, dtype=np.float32)
    alt_node = np.full((P, n_alt), -1, dtype=np.int32)
    alt_score = np.full((P, n_alt), -np.inf, dtype=np.float32)
    for g, X in enumerate(G):
        if status[g] == 2:
            continue
        L = levels[g]
        excl = bool(X.flags & lw.STEP_EXCLUSIVE)
        own = level_owner(dom, owner, n_domains, L, last, pods) if excl else None
        for w, wave in enumerate(X.waves):
            for p, (ri, first, reps) in enumerate(wave):
                if (g, w, p) not in rows:
                    continue
                row = rows[(g, w, p)]
                part = excl and bool(X.rflags[ri] & lw.ROLE_EXCLUSIVE)
                emask = ((dom[L] == domain[g]) & ((own == FREE) | (own == X.gid))) if part else None
                cdom = dom[X.C[ri]] if X.C[ri] >= 0 else None
                base = X.pod0 + X.first_pod[ri] + first * X.S[ri]
                for pod in range(base, base + reps * X.S[ri]):
                    node = int(assign[pod])
                    if node < 0:
                        continue
                    ok = ranked_candidates(row, node, free, used, X.demand[ri], emask, cdom)
                    idx = np.nonzero(ok)[0]
                    best = idx[np.lexsort((idx, -row[idx].astype(np.float64)))][:n_alt]
                    score[pod] = row[node]
                    alt_node[pod, :len(best)] = best
                    alt_score[pod, :len(best)] = row[best]
    return assign, status, domain, score, alt_node, alt_score
