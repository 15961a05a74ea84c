"""Oracle of ranked alternates for committed leader-worker batches (rbgtopo_place_groups_lw_committed_ranked,
DESIGN.md §3.15; test infrastructure, built on tests/lw_committed_oracle.py without restating its loop).

`run_lw_committed_rows` runs lw_committed_oracle.run_lw_committed and keeps the dense row of every (group, wave, role)
as that group's run scored it: the rows are taken where run_group hands them to lw_oracle.place_wave (wrapped for the
duration of the call).  The oracle places each group once, in blob order, so these are the rows of every group's
final run.  §3.15 is then applied in numpy, the way tests/committed_alternates_oracle.py applies §3.14 and
tests/lw_alternates_oracle.py applies §3.12:
  * used_B[n]: the demand of every pod the batch placed on n (a failed gang places nothing);
  * own_B,g: the level-0 owner a group placed after the whole batch would see — the snapshot's domain owner with the
    last reporter of every domain applied (map mode), or merge_claims(owner0, last reporter) (occupancy mode);
  * candidates of placed pod p of role rho: S_p[n] != -inf, n != assign[p], free[n] - used_B[n] >= demand_rho, for a
    participating role of an exclusive group dom_0(n) = domain[g] and own_B,g[n] in {-1, gid_g}, and for a role with
    C >= 0 dom_C(n) = dom_C(assign[p]); ranked by score descending, node ascending."""
from __future__ import annotations

from typing import Optional

import numpy as np

import lw_committed_oracle as lco
import lw_oracle as lw
from committed_oracle import FREE, merge_claims
from lw_alternates_oracle import ranked_candidates


def run_lw_committed_rows(topo, gblob, role_pods, **kw):
    """lw_committed_oracle.run_lw_committed(topo, gblob, role_pods, **kw) plus rows[(g, w, p)]: the dense row of group
    g's wave w, role row p.  A group with pods is known by its first pod, which no other such group shares."""
    first_pod = {X.pod0: g for g, X in enumerate(lco.groups_of(gblob, role_pods)) if X.n_pods}
    rows = {}
    inner = lw.place_wave

    def keep(G, w, wave_rows, *args):
        for p, row in enumerate(wave_rows):
            rows[(first_pod[G.pod0], w, p)] = np.array(row, dtype=np.float32, copy=True)
        return inner(G, w, wave_rows, *args)

    lw.place_wave = keep
    try:
        out = lco.run_lw_committed(topo, gblob, role_pods, **kw)
    finally:
        lw.place_wave = inner
    return (*out, rows)


def run_lw_committed_ranked(topo, gblob, role_pods, n_alt: int, level_domain=None,
                            owner0: Optional[np.ndarray] = None):
    """(assign, status, domain, score[P], alt_node[P, n_alt], alt_score[P, n_alt]); arguments as
    lw_committed_oracle.run_lw_committed (owner0: occupancy mode)."""
    assign, status, domain, rows = run_lw_committed_rows(topo, gblob, role_pods, level_domain=level_domain,
                                                         owner0=owner0)
    level_domain = [topo.domain] if level_domain is None else level_domain
    dom0 = np.asarray(topo.domain, dtype=np.int64)
    free = np.asarray(topo.free, dtype=np.int64)
    G = lco.groups_of(gblob, role_pods)
    used = np.zeros(len(free), dtype=np.int64)
    last = np.full(len(topo.domain_owner), FREE, np.int32)   # the last reporter of every level-0 domain
    for g, X in enumerate(G):
        for ri in range(X.q):
            first = X.pod0 + X.first_pod[ri]
            for node in assign[first:first + X.pending[ri] * X.S[ri]]:
                if node >= 0:
                    used[node] += X.demand[ri]
        if (X.flags & lw.STEP_EXCLUSIVE) and status[g] != 2 and domain[g] >= 0:
            last[domain[g]] = X.gid
    if owner0 is not None:
        own = merge_claims(np.asarray(owner0, dtype=np.int32), last[dom0])
    else:
        own = np.array(topo.domain_owner, dtype=np.int32, copy=True)
        own[last != FREE] = last[last != FREE]
        own = own[dom0]
    P = len(assign)
    score = np.full(P, -np.inf, dtype=np.float32)
    alt_node = np.full((P, n_alt), -1, dtype=np.int32)
    alt_score = np.full((P, n_alt), -np.inf, dtype=np.float32)
    for g, X in enumerate(G):
        if status[g] == 2:   # gang failed: nothing of the group is placed
            continue
        excl = bool(X.flags & lw.STEP_EXCLUSIVE)
        for w, wave in enumerate(X.waves):
            for p, (ri, first, reps) in enumerate(wave):
                if (g, w, p) not in rows:
                    continue
                row = rows[(g, w, p)]
                part = excl and bool(X.rflags[ri] & lw.ROLE_EXCLUSIVE)
                emask = ((dom0 == domain[g]) & ((own == FREE) | (own == X.gid))) if part else None
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
