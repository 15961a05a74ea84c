"""The snapshot one exclusive group sees at its level L (DESIGN.md §3.9; test infrastructure).

levels_oracle.group_view generalised from level 0 to any level: domain' = 2·dom_L(n) + blocked_g(n) with blocked from
owner_L, owner'[2d] = -1 and owner'[2d + 1] = another gid.  Feasibility per node is that of owner_L, D* (the domain of
the best feasible node, never blocked) is always even, so fixed' = 2·fixed and the reported domain is domain' // 2:
oracle/wave_loop.py places the group unchanged.
"""
from __future__ import annotations

import numpy as np

import levels_oracle as lo
from oracle import wave_loop
from rbg_b200 import synth


def level_view(topo: synth.Topology, level_domain: np.ndarray, owner: np.ndarray, n_domains, level: int, gid: int,
               other_gid: int) -> synth.Topology:
    """level_domain / owner: [n_levels + 1][n] (row 0 = level 0); n_domains: domain count per level."""
    assert other_gid != gid
    blocked = ~((owner[level] == lo.FREE) | (owner[level] == gid))
    dom = 2 * np.asarray(level_domain[level], dtype=np.int64) + blocked
    own = np.full(2 * int(n_domains[level]), lo.FREE, dtype=np.int32)
    own[1::2] = other_gid
    return synth.Topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free.copy(), dom.astype(np.int32), own)


def with_levels(gblob: np.ndarray, levels) -> np.ndarray:
    """The GROUPS blob with group g's exclusive level (word +10) set to levels[g]."""
    b = np.array(gblob, dtype=np.int32, copy=True)
    for g, L in enumerate(levels):
        b[8 + 12 * g + 10] = L
    return b


def expected_fleet(topo, level_domain, owner, n_domains, gblob):
    """Per group (assign in group order, status, domain) of the wave loop on the group's level view, plus the views."""
    ng = int(gblob[2])
    gids = [int(gblob[8 + 12 * g]) for g in range(ng)]
    other = lo.unused_gid(gids)
    out, views = [], []
    for g in range(ng):
        L = int(gblob[8 + 12 * g + 10])
        view = level_view(topo, level_domain, owner, n_domains, L, gids[g], other)
        states, _ = wave_loop.run_fleet(view, wave_loop.groups_from_blob(lo.groups_blob_for_view(gblob, g)))
        r = states[g].result()
        out.append((states[g].assign_in_group_order(), r["status"], r["domain"] // 2 if r["domain"] >= 0 else -1))
        views.append(view)
    return out, views
