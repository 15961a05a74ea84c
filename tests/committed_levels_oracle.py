"""Oracle of the committed batch at exclusive levels (DESIGN.md §3.8 / §3.9).  TEST INFRASTRUCTURE, a sibling of
tests/committed_oracle.py built on the same pieces (its run_group / group_claims / merge_claims, levels_oracle and
levels_view): it never imports rbg_b200's native code.

`run_fleet_committed_levels(topo, groups, group_levels, level_domain, owner, n_domains)` places the groups one after
another in the given order (occupancy mode), group g at its exclusive level L_g:
  * capacity: as in run_fleet_committed, every placed replica of an earlier group is consumed (node, demand);
  * ownership: group g sees levels_view.level_view of owner_g = owner_{L_g} ⊕ K ⊕ P (`level_owner`), where K merges,
    for every level L, the gid of the last earlier exclusive reporter (status != 2) of dom_L(n) at level L, and P the gid
    of every placed participating replica of an earlier exclusive group keyed at another level, in dom_{L_g}(n).
For a batch whose groups are all at level 0 this is run_fleet_committed(owner0=owner[0])
(tests/test_oracle_committed_levels.py checks it)."""
from __future__ import annotations

import copy
from typing import Dict, List, Optional, Sequence

import numpy as np

import levels_oracle
import levels_view
from committed_oracle import group_claims, merge_claims, run_group
from oracle import wave_loop

FREE = levels_oracle.FREE


def participating_pods(s: wave_loop.GroupState) -> List[int]:
    """Nodes of the placed replicas of the group's participating (exclusive) roles; none for a failed gang."""
    nodes = s.result()["nodes"]
    out = []
    for ri in s.order:
        if not s.g.roles[ri].exclusive:
            continue
        for c in range(s.pending[ri]):
            m = nodes[f"{s.g.name}-{s.g.roles[ri].name}-{s.first[ri] + c}"]
            if m >= 0:
                out.append(m)
    return out


def level_owner(level_domain: np.ndarray, owner: np.ndarray, n_domains, level: int, last, pods) -> np.ndarray:
    """owner_g[n] of a group at `level`: owner_level[n] ⊕ K(n) ⊕ P(n), with last[L][d] = the gid of the last earlier
    exclusive reporter of domain d of level L (-1 = none) and pods = (gid, level of its group, node) of every placed
    participating replica of an earlier exclusive group."""
    dom = np.asarray(level_domain)
    own = np.asarray(owner[level], dtype=np.int32)
    for L in range(dom.shape[0]):                                   # K: the earlier groups' domains, at their level
        own = merge_claims(own, last[L][dom[L]])
    pd = np.full(int(n_domains[level]), FREE, np.int32)             # P: pods keyed elsewhere, in this group's domain
    for gid, lh, m in pods:
        if lh != level:
            d = int(dom[level, m])
            pd[d] = levels_oracle.merge(int(pd[d]), gid)
    return merge_claims(own, pd[dom[level]])


def run_fleet_committed_levels(topo, groups: Sequence[wave_loop.OGroup], group_levels: Sequence[int],
                               level_domain: np.ndarray, owner: np.ndarray, n_domains, nthreads: int = 1,
                               limit: Optional[int] = None, fast: bool = False, terms: Sequence[str] = ("K", "P"),
                               reporter: str = "last") -> List[wave_loop.GroupState]:
    """States in the given order.  level_domain [n_levels + 1][n] (row 0 = the snapshot's domain), owner =
    levels_oracle.derive_level_owner(level_domain, occ), n_domains per level.  `limit`: place only the first `limit`
    groups.  `terms` and `reporter` exist for the preconditions of tests/commit_levels_limits_cases.py: the owner
    without the domain term K or the pod term P, or with the first earlier reporter of a domain instead of the last."""
    assert set(terms) <= {"K", "P"} and reporter in ("last", "first")
    dom = np.asarray(level_domain)
    last = [np.full(int(n_domains[L]), FREE, np.int32) for L in range(dom.shape[0])]
    pods: List = []
    claimed: Dict[int, int] = {}
    gids = {g.gid for g in groups}
    other = levels_oracle.unused_gid(gids)          # a gid of no group that fits int32 (gids reach 2^31 - 1)
    states: List = []
    for g, L in zip(groups[:limit], group_levels):
        ow = np.array(owner, dtype=np.int32, copy=True)
        ow[L] = level_owner(dom, owner, n_domains, L, last, pods)
        t = levels_view.level_view(topo, dom, ow, n_domains, L, g.gid, other)
        gv = copy.copy(g)   # the view numbers domain d of level L as 2d (2d + 1 for its nodes blocked to g)
        gv.fixed_domain = 2 * g.fixed_domain if g.fixed_domain >= 0 else g.fixed_domain
        s = run_group(t, gv, claimed, nthreads, fast)
        s.g = g
        if s.fixed_domain >= 0:
            s.fixed_domain //= 2
        for node, amt in group_claims(s).items():
            claimed[node] = claimed.get(node, 0) + amt
        res = s.result()
        if g.exclusive and res["status"] != 2:
            if res["domain"] >= 0 and "K" in terms and (reporter == "last" or last[L][res["domain"]] == FREE):
                last[L][res["domain"]] = g.gid
            if "P" in terms:
                pods += [(g.gid, L, m) for m in participating_pods(s)]
        states.append(s)
    return states


def group_levels(gblob) -> List[int]:
    """Word +10 (exclusive level) of every group record."""
    return [int(gblob[8 + 12 * g + 10]) for g in range(int(gblob[2]))]
