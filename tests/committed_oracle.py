"""Oracle of the committed batch (DESIGN.md §3.8).  TEST INFRASTRUCTURE, built only on the oracle package
(oracle/wave_loop.py, oracle/placer.py): it never imports rbg_b200.

`run_fleet_committed(topo, groups)` places the groups one after another in the given order, each through the
oracle's own level / wave loop (`wave_loop.GroupState`, exact `need` from the replicas actually unplaced):
  * group g starts with `consumed` = the capacity the placed replicas of every earlier group took, (node, demand)
    per replica; a gang-failed group takes nothing;
  * group g sees a copy of the snapshot whose domain_owner carries the exclusive domains the earlier groups
    reported (status != 2, domain >= 0), owned by the reporting group's gid."""
from __future__ import annotations

import copy
from typing import Dict, List, Optional, Sequence

import numpy as np

from oracle import placer as oracle_placer
from oracle import wave_loop


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


def run_group(topo, g: wave_loop.OGroup, consumed: Dict[int, int], nthreads: int = 1) -> wave_loop.GroupState:
    """One group through its wave loop against `topo`, with `consumed` capacity already taken."""
    s = wave_loop.GroupState(g)
    s.consumed = dict(consumed)
    for w in range(len(s.waves)):
        if s.failed:
            break
        r = oracle_placer.place(topo, wave_loop.build_blob([s.step(w)]), want_matrix=False, want_topk=False,
                                nthreads=nthreads)
        if r["rc"] != 0:
            raise RuntimeError(f"oracle rc={r['rc']} in wave {w} of {g.name}")
        s.absorb(w, r["assign"], int(r["status"][0]), int(r["domain"][0]))
    return s


def run_fleet_committed(topo, groups: Sequence[wave_loop.OGroup], nthreads: int = 1,
                        limit: Optional[int] = None) -> List[wave_loop.GroupState]:
    """The committed batch, states in the given order.  `limit`: place only the first `limit` groups (they do not
    depend on the groups after them)."""
    owner = np.array(topo.domain_owner, dtype=np.int32, copy=True)
    claimed: Dict[int, int] = {}
    states: List = []
    for g in groups[:limit]:
        t = copy.copy(topo)
        t.domain_owner = owner.copy()
        s = run_group(t, g, claimed, nthreads)
        for node, amt in group_claims(s).items():
            claimed[node] = claimed.get(node, 0) + amt
        res = s.result()
        if g.exclusive and res["status"] != 2 and res["domain"] >= 0:
            owner[res["domain"]] = g.gid
        states.append(s)
    return states


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
