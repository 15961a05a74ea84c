"""Oracle of the committed batch (DESIGN.md §3.8).  TEST INFRASTRUCTURE, built only on the oracle package
(oracle/wave_loop.py, oracle/placer.py): it never imports rbg_b200.

`run_fleet_committed(topo, groups)` places the groups one after another in the given order, each through the
oracle's own level / wave loop (`wave_loop.GroupState`, exact `need` from the replicas actually unplaced):
  * group g starts with `consumed` = the capacity the placed replicas of every earlier group took, (node, demand)
    per replica; a gang-failed group takes nothing;
  * group g sees a copy of the snapshot whose domain_owner carries the exclusive domains the earlier groups
    reported (status != 2, domain >= 0), owned by the reporting group's gid;
  * occupancy mode (DESIGN.md §3.9, `owner0` = the derived level-0 owner of every node): group g sees
    levels_oracle.group_view of merge(owner0[n], gid of the last earlier reporter of the level-0 domain of n) — a
    claim is merged into the owner the records derive, it never replaces it.
`fast` runs every wave through oracle_placer.place_fast, which tests/test_oracle_fast.py bit-checks against the
literal oracle (and tests/test_oracle_committed.py the committed loop on top of it)."""
from __future__ import annotations

import copy
from typing import Dict, List, Optional, Sequence

import numpy as np

import levels_oracle
from oracle import placer as oracle_placer
from oracle import wave_loop

FREE, BLOCKED = levels_oracle.FREE, levels_oracle.BLOCKED


def group_claims(s: wave_loop.GroupState) -> Dict[int, int]:
    """node -> capacity the group's placed replicas take (empty for a failed gang)."""
    res = s.result()
    out: Dict[int, int] = {}
    for wave in s.waves:
        for ri, ordinal, cnt in wave:
            for c in range(cnt):
                node = res["nodes"][f"{s.g.name}-{s.g.roles[ri].name}-{ordinal + c}"]
                if node >= 0:
                    out[node] = out.get(node, 0) + s.g.roles[ri].demand
    return out


def run_group(topo, g: wave_loop.OGroup, consumed: Dict[int, int], nthreads: int = 1,
              fast: bool = False) -> wave_loop.GroupState:
    """One group through its wave loop against `topo`, with `consumed` capacity already taken."""
    place = oracle_placer.place_fast if fast else oracle_placer.place
    s = wave_loop.GroupState(g)
    s.consumed = dict(consumed)
    for w in range(len(s.waves)):
        if s.failed:
            break
        r = place(topo, wave_loop.build_blob([s.step(w)]), want_matrix=False, want_topk=False, nthreads=nthreads)
        if r["rc"] != 0:
            raise RuntimeError(f"oracle rc={r['rc']} in wave {w} of {g.name}")
        s.absorb(w, r["assign"], int(r["status"][0]), int(r["domain"][0]))
    return s


def run_fleet_committed(topo, groups: Sequence[wave_loop.OGroup], nthreads: int = 1, limit: Optional[int] = None,
                        owner0: Optional[np.ndarray] = None, fast: bool = False) -> List[wave_loop.GroupState]:
    """The committed batch, states in the given order.  `limit`: place only the first `limit` groups (they do not
    depend on the groups after them).  `owner0`: occupancy mode; the snapshot's domain_owner is then not read."""
    occ = owner0 is not None
    # domain -> the owner group g sees: the snapshot's map with the claims, or (occupancy mode) the claims alone
    owner = np.full(len(topo.domain_owner), FREE, np.int32) if occ else np.array(topo.domain_owner, np.int32, copy=True)
    claimed: Dict[int, int] = {}
    states: List = []
    for g in groups[:limit]:
        if not occ:
            t = copy.copy(topo)
            t.domain_owner = owner.copy()
            s = run_group(t, g, claimed, nthreads, fast)
        else:   # the view numbers domain d as 2d (2d + 1 for its nodes blocked to g)
            t = levels_oracle.group_view(topo, merge_claims(np.asarray(owner0), owner[topo.domain]), g.gid, g.gid + 1)
            gv = copy.copy(g)
            gv.fixed_domain = 2 * g.fixed_domain if g.fixed_domain >= 0 else g.fixed_domain
            s = run_group(t, gv, claimed, nthreads, fast)
            s.g = g
            if s.fixed_domain >= 0:
                s.fixed_domain //= 2
        for node, amt in group_claims(s).items():
            claimed[node] = claimed.get(node, 0) + amt
        res = s.result()
        if g.exclusive and res["status"] != 2 and res["domain"] >= 0:
            owner[res["domain"]] = g.gid
        states.append(s)
    return states


def merge_claims(owner0: np.ndarray, claim: np.ndarray) -> np.ndarray:
    """levels_oracle.merge element-wise: the derived owner of every node with the gid of the last earlier reporter of
    its domain (-1 = none)."""
    return np.where(claim == FREE, owner0,
                    np.where((owner0 == FREE) | (owner0 == claim), claim, BLOCKED)).astype(np.int32)


def run_fleet_snapshot(topo, groups: Sequence[wave_loop.OGroup], nthreads: int = 1) -> List[wave_loop.GroupState]:
    """Snapshot semantics (DESIGN.md §3.7): every group against the same snapshot."""
    states, _ = wave_loop.run_fleet(topo, groups, nthreads=nthreads)
    return states


def result_arrays(states):
    """(assign in GROUPS-blob order, status, domain) of a list of states."""
    a: List[int] = []
    st, dm = [], []
    for s in states:
        a.extend(s.assign_in_group_order())
        r = s.result()
        st.append(r["status"])
        dm.append(r["domain"])
    return np.asarray(a, dtype=np.int32), np.asarray(st, dtype=np.int32), np.asarray(dm, dtype=np.int32)
