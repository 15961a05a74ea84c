"""Oracle of ranked alternates for leader-worker pods (rbgtopo_place_groups_lw_ranked, DESIGN.md §3.12; test
infrastructure).

tests/lw_oracle.run_lw places the pods; run_lw_rows keeps the dense row of every (wave, role) it placed from, as
lw_oracle.place_wave receives them, without restating the loop.  §3.12 is then applied in numpy, the way
tests/alternates_oracle.py applies §3.10.  The candidates of
placed pod p of role rho are the nodes n with S_p[n] != -inf, n != assign[p], free[n] - used_g[n] >= demand_rho
(used_g: the demand of every placed pod of the group on n), dom_{L_g}(n) = domain[g] for a participating role of an
exclusive group, and dom_C(n) = dom_C(assign[p]) for a role with C >= 0; they are ranked by score descending, node
ascending.  score[p] = S_p[assign[p]]; unplaced pods and every pod of a gang-failed group get -inf and no alternates."""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np

import lw_oracle as lw


def groups_of(gblob, role_pods):
    """The LwGroup of every group in blob order (waves, S, C, first pods), as run_lw builds them."""
    gb = np.asarray(gblob, dtype=np.int64)
    rp = np.asarray(role_pods, dtype=np.int64).reshape(-1, 2)
    out, r0, pod0 = [], 0, 0
    for g in range(int(gb[2])):
        q = int(gb[lw.HDR + lw.GW * g + 3])
        out.append(lw.LwGroup(gb, g, rp[r0:r0 + q], pod0))
        r0 += q
        pod0 += out[-1].n_pods
    return out


def run_lw_rows(topo, gblob, role_pods, **kw):
    """lw_oracle.run_lw(topo, gblob, role_pods, **kw) plus rows[(g, w, p)]: the dense row of group g's wave w, role p.
    The rows are taken where run_lw hands them to lw_oracle.place_wave (wrapped for the duration of the call); a group
    with pods is known by its first pod, which no other such group shares."""
    first_pod = {X.pod0: g for g, X in enumerate(groups_of(gblob, role_pods)) if X.n_pods}
    rows = {}
    inner = lw.place_wave

    def keep(G, w, wave_rows, *args):
        for p, row in enumerate(wave_rows):
            rows[(first_pod[G.pod0], w, p)] = np.array(row, dtype=np.float32, copy=True)
        return inner(G, w, wave_rows, *args)

    lw.place_wave = keep
    try:
        out = lw.run_lw(topo, gblob, role_pods, **kw)
    finally:
        lw.place_wave = inner
    return (*out, rows)


def ranked_candidates(row, node, free, used, demand, excl_mask, coloc_dom):
    """Boolean mask of the §3.12 candidates of a pod on `node` reading `row`."""
    ok = (row != -np.inf) & (free - used >= demand)
    ok[node] = False
    if excl_mask is not None:
        ok &= excl_mask
    if coloc_dom is not None:
        ok &= coloc_dom == coloc_dom[node]
    return ok


def run_lw_ranked(topo, gblob, role_pods, n_alt: int, level_domain=None, excl_domain=None,
                  groups: Optional[Sequence[int]] = None):
    """(assign, status, domain, score[P], alt_node[P, n_alt], alt_score[P, n_alt]); arguments as lw_oracle.run_lw.
    Groups left out keep run_lw's -1 / -9 / -9 and score -inf without alternates."""
    assign, status, domain, rows = run_lw_rows(topo, gblob, role_pods, level_domain=level_domain,
                                               excl_domain=excl_domain, groups=groups)
    level_domain = [topo.domain] if level_domain is None else level_domain
    excl_domain = np.asarray(topo.domain if excl_domain is None else excl_domain)
    free = np.asarray(topo.free, dtype=np.int64)
    P = len(assign)
    score = np.full(P, -np.inf, dtype=np.float32)
    alt_node = np.full((P, n_alt), -1, dtype=np.int32)
    alt_score = np.full((P, n_alt), -np.inf, dtype=np.float32)
    G = groups_of(gblob, role_pods)
    for g in (range(len(G)) if groups is None else groups):
        X = G[g]
        if status[g] == 2:   # gang failed: nothing of the group is placed
            continue
        used = np.zeros(len(free), dtype=np.int64)
        for ri in range(X.q):
            first = X.pod0 + X.first_pod[ri]
            for node in assign[first:first + X.pending[ri] * X.S[ri]]:
                if node >= 0:
                    used[node] += X.demand[ri]
        excl = bool(X.flags & lw.STEP_EXCLUSIVE)
        for w, wave in enumerate(X.waves):
            for p, (ri, first, reps) in enumerate(wave):
                if (g, w, p) not in rows:
                    continue
                row = rows[(g, w, p)]
                part = excl and bool(X.rflags[ri] & lw.ROLE_EXCLUSIVE)
                emask = (excl_domain == domain[g]) if part else None
                cdom = np.asarray(level_domain[X.C[ri]]) if X.C[ri] >= 0 else None
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
