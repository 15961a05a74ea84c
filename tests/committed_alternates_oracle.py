"""Oracle of ranked alternates for committed batches (rbgtopo_place_groups_committed_ranked, DESIGN.md §3.14; test
infrastructure, built on the committed oracles without restating their loops).

`run_committed_rows` runs committed_oracle.run_fleet_committed (map or occupancy mode) or
committed_levels_oracle.run_fleet_committed_levels (levels) and keeps the dense row of every replica's wave as that
group's committed wave loop scored it: the rows are taken where the loop hands a wave's result to
wave_loop.GroupState.absorb, with the oracle scorer asked for its matrix (both wrapped for the duration of the call).
The views of the occupancy and level oracles number domains 2d / 2d + 1 but keep one row entry per node, so the rows
are used as they are.  §3.14 is then applied in numpy:
  * used_B[n]: the demand of every replica the batch placed on n (a failed gang places nothing);
  * own_B,g: the owner a group of gid_g placed after the whole batch would see — the snapshot's domain owner with the
    last reporter of every domain applied (map mode), merge_claims(owner0, last reporter) (occupancy mode), or
    level_owner(..., last, pods) at L_g over every group of the batch (levels);
  * candidates of placed replica r: S_r[n] != -inf, n != assign[r], free[n] - used_B[n] >= demand, and for a
    participating role of an exclusive group dom_{L_g}(n) = domain[g] and own_B,g[n] in {-1, gid_g}; ranked by score
    descending, node ascending."""
from __future__ import annotations

from typing import Dict, Optional, Sequence

import numpy as np

import committed_levels_oracle as clo
import committed_oracle as co
import levels_oracle
from oracle import placer as oracle_placer
from oracle import wave_loop

FREE = levels_oracle.FREE


def _key(g: wave_loop.OGroup, ri: int, ordinal: int) -> str:
    return f"{g.name}-{g.roles[ri].name}-{ordinal}"


def run_committed_rows(topo, groups: Sequence[wave_loop.OGroup], owner0: Optional[np.ndarray] = None,
                       levels: Optional[dict] = None, fast: bool = False):
    """(states, rows): the committed oracle's states and rows[replica key] = the dense row its wave was placed from.
    levels: dict(group_levels, level_domain, owner, n_domains) for run_fleet_committed_levels, else
    run_fleet_committed(owner0=owner0)."""
    rows: Dict[str, np.ndarray] = {}
    last = {}
    inner_place, inner_state = oracle_placer.place, wave_loop.GroupState

    def place(topo_, blob, *args, **kw):  # place_fast calls it too, with its arguments positional
        if args:
            args = (True,) + args[1:]
        else:
            kw["want_matrix"] = True
        r = inner_place(topo_, blob, *args, **kw)
        last["matrix"] = r["matrix"]
        return r

    class KeptState(inner_state):
        def absorb(self, w, assign, status, domain):
            off = 0
            for ri, ordinal, cnt in self.waves[w]:
                row = np.array(last["matrix"][off], dtype=np.float32, copy=True)
                for c in range(cnt):
                    rows[_key(self.g, ri, ordinal + c)] = row
                off += cnt
            return super().absorb(w, assign, status, domain)

    oracle_placer.place = place
    wave_loop.GroupState = KeptState
    try:
        if levels is None:
            states = co.run_fleet_committed(topo, groups, owner0=owner0, fast=fast)
        else:
            states = clo.run_fleet_committed_levels(topo, groups, levels["group_levels"], levels["level_domain"],
                                                    levels["owner"], levels["n_domains"], fast=fast)
    finally:
        oracle_placer.place, wave_loop.GroupState = inner_place, inner_state
    return states, rows


def run_fleet_committed_ranked(topo, groups: Sequence[wave_loop.OGroup], n_alt: int,
                               owner0: Optional[np.ndarray] = None, levels: Optional[dict] = None,
                               fast: bool = False):
    """(assign, status, domain, score[R], alt_node[R, n_alt], alt_score[R, n_alt]) in GROUPS-blob order."""
    states, rows = run_committed_rows(topo, groups, owner0=owner0, levels=levels, fast=fast)
    n = len(topo.free)
    free = np.asarray(topo.free, dtype=np.int64)
    used = np.zeros(n, dtype=np.int64)
    for s in states:
        for node, amt in co.group_claims(s).items():
            used[node] += amt
    # the last reporter of every domain over the whole batch, and (levels) every participating pod
    if levels is None:
        dom_g = [np.asarray(topo.domain, dtype=np.int64)]
        last = [np.full(len(topo.domain_owner), FREE, np.int32)]
        lv = [0] * len(states)
    else:
        dom_g = [np.asarray(x, dtype=np.int64) for x in levels["level_domain"]]
        last = [np.full(int(k), FREE, np.int32) for k in levels["n_domains"]]
        lv = list(levels["group_levels"])
    pods = []
    for s, L in zip(states, lv):
        res = s.result()
        if s.g.exclusive and res["status"] != 2:
            if res["domain"] >= 0:
                last[L][res["domain"]] = s.g.gid
            pods += [(s.g.gid, L, m) for m in clo.participating_pods(s)]

    def owner_after(L: int) -> np.ndarray:
        if levels is not None:
            return clo.level_owner(levels["level_domain"], levels["owner"], levels["n_domains"], L, last, pods)
        if owner0 is not None:
            return co.merge_claims(np.asarray(owner0, dtype=np.int32), last[0][dom_g[0]])
        own = np.array(topo.domain_owner, dtype=np.int32, copy=True)
        own[last[0] != FREE] = last[0][last[0] != FREE]
        return own[dom_g[0]]

    assign, status, dom_out, score, alt_node, alt_score = [], [], [], [], [], []
    for s, L in zip(states, lv):
        res = s.result()
        status.append(res["status"])
        dom_out.append(res["domain"])
        own = owner_after(L) if s.g.exclusive else None
        for ri in s.order:
            role = s.g.roles[ri]
            for c in range(s.pending[ri]):
                k = _key(s.g, ri, s.first[ri] + c)
                node = res["nodes"][k]
                assign.append(node)
                if node < 0:
                    score.append(-np.inf)
                    alt_node.append([-1] * n_alt)
                    alt_score.append([-np.inf] * n_alt)
                    continue
                S = rows[k]
                ok = (S != -np.inf) & (free - used >= role.demand)
                ok[node] = False
                if s.g.exclusive and role.exclusive:
                    ok &= (dom_g[L] == res["domain"]) & ((own == FREE) | (own == s.g.gid))
                idx = np.nonzero(ok)[0]
                best = idx[np.lexsort((idx, -S[idx].astype(np.float64)))][:n_alt]
                score.append(float(S[node]))
                alt_node.append([int(x) for x in best] + [-1] * (n_alt - len(best)))
                alt_score.append([float(S[x]) for x in best] + [-np.inf] * (n_alt - len(best)))
    R = len(assign)
    return (np.asarray(assign, dtype=np.int32), np.asarray(status, dtype=np.int32), np.asarray(dom_out, dtype=np.int32),
            np.asarray(score, dtype=np.float32), np.asarray(alt_node, dtype=np.int32).reshape(R, n_alt),
            np.asarray(alt_score, dtype=np.float32).reshape(R, n_alt))
