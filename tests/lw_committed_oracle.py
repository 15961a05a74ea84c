"""Oracle of the committed leader-worker batch (rbgtopo_place_groups_lw_committed, DESIGN.md §3.13; test
infrastructure, built on tests/lw_oracle.py and tests/committed_oracle.py: it never imports rbg_b200).

The groups are placed one after another in blob order.  Group g runs the §3.11 loop of lw_oracle (`LwGroup`,
`place_wave` on the oracle scorer's dense rows) alone, with
  * `consumed` seeded with (node, demand) of every pod an earlier group placed (a gang-failed group takes nothing);
  * the owners committed_oracle gives it: a copy of the snapshot whose domain_owner carries the exclusive domains the
    earlier groups reported (status != 2, domain >= 0; the last reporter wins), or in occupancy mode (`owner0`, the
    derived level-0 owner of every node) levels_oracle.group_view of merge_claims(owner0, claims).
In the occupancy view domain d is numbered 2d (2d + 1 for its nodes blocked to g); co-location at level 0 still reads
the snapshot's own domain[], so `level_domain` is always the caller's partitions."""
from __future__ import annotations

import copy
from typing import Dict, List, Optional

import numpy as np

import levels_oracle
import lw_oracle as lw
from committed_oracle import FREE, merge_claims
from oracle import placer as oracle_placer
from oracle import wave_loop


def run_group(topo, X: lw.LwGroup, level_domain, excl_domain, assign: np.ndarray) -> None:
    """The §3.11 loop of one group against `topo` (X.consumed already holds what earlier groups took)."""
    for w in range(len(X.waves)):
        if X.failed:
            break
        r = oracle_placer.place(topo, wave_loop.build_blob([X.step(w)]), want_matrix=True, want_topk=False)
        if r["rc"] != 0:
            raise RuntimeError(f"oracle rc={r['rc']} in wave {w} of group gid {X.gid}")
        rows, k = [], 0
        for ri, _, reps in X.waves[w]:
            rows.append(r["matrix"][k])
            k += reps * X.S[ri]
        pods, st, dstar = lw.place_wave(X, w, rows, topo, excl_domain, level_domain)
        i, any_placed = 0, False
        for ri, first, reps in X.waves[w]:
            base = X.pod0 + X.first_pod[ri] + first * X.S[ri]
            for j in range(reps * X.S[ri]):
                node = pods[i]
                i += 1
                assign[base + j] = node
                if node >= 0:
                    any_placed = True
                    X.anchors[(node, ri)] = X.anchors.get((node, ri), 0) + 1
                    X.consumed[node] = X.consumed.get(node, 0) + X.demand[ri]
                    X.unplaced[ri] -= 1
        if (X.flags & lw.STEP_EXCLUSIVE) and dstar >= 0 and any_placed:
            X.fixed = dstar
        X.status = max(X.status, st)
        if (X.flags & lw.STEP_GANG) and st != 0:
            X.failed = True


def groups_of(gblob, role_pods) -> List[lw.LwGroup]:
    gb = np.asarray(gblob, dtype=np.int64)
    rp = np.asarray(role_pods, dtype=np.int64).reshape(-1, 2)
    out: List[lw.LwGroup] = []
    r0 = pod0 = 0
    for g in range(int(gb[2])):
        q = int(gb[lw.HDR + lw.GW * g + 3])
        out.append(lw.LwGroup(gb, g, rp[r0:r0 + q], pod0))
        r0 += q
        pod0 += out[-1].n_pods
    return out


def run_lw_committed(topo, gblob, role_pods, level_domain=None, owner0: Optional[np.ndarray] = None,
                     limit: Optional[int] = None):
    """The committed batch.  level_domain: the partitions co-location level C indexes (default [topo.domain]);
    owner0: occupancy mode, the snapshot's domain_owner is then not read; limit: place only the first `limit` groups
    (they do not depend on the later ones).  Returns (assign per pod, status[ng], domain[ng]); groups past `limit`
    keep -1 / -9 / -9."""
    G = groups_of(gblob, role_pods)
    ng = len(G)
    level_domain = [topo.domain] if level_domain is None else level_domain
    n_pods = sum(X.n_pods for X in G)
    assign = np.full(n_pods, -1, dtype=np.int32)
    status = np.full(ng, -9, dtype=np.int32)
    domain = np.full(ng, -9, dtype=np.int32)
    occ = owner0 is not None
    owner = np.full(len(topo.domain_owner), FREE, np.int32) if occ else np.array(topo.domain_owner, np.int32, copy=True)
    claimed: Dict[int, int] = {}
    for g in range(ng if limit is None else min(limit, ng)):
        X = G[g]
        X.consumed = dict(claimed)
        if not occ:
            t = copy.copy(topo)
            t.domain_owner = owner.copy()
            run_group(t, X, level_domain, topo.domain, assign)
        else:
            t = levels_oracle.group_view(topo, merge_claims(np.asarray(owner0), owner[topo.domain]), X.gid, X.gid + 1)
            if X.fixed >= 0:
                X.fixed *= 2
            run_group(t, X, level_domain, t.domain, assign)
            if X.fixed >= 0:
                X.fixed //= 2
        excl = bool(X.flags & lw.STEP_EXCLUSIVE)
        if X.failed:
            assign[X.pod0:X.pod0 + X.n_pods] = -1
            status[g], domain[g] = 2, -1
            continue
        status[g] = X.status
        domain[g] = X.fixed if excl else -1
        for ri in range(X.q):
            lo = X.pod0 + X.first_pod[ri]
            for node in assign[lo:lo + X.pending[ri] * X.S[ri]]:
                if node >= 0:
                    claimed[int(node)] = claimed.get(int(node), 0) + X.demand[ri]
        if excl and domain[g] >= 0:
            owner[domain[g]] = X.gid
    return assign, status, domain
