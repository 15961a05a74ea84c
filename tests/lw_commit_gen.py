"""Committed leader-worker batches for the tests (DESIGN.md §3.13): seeded fleets of multi-pod groups with mixed
(S, C), exclusive and gang groups, shared gids, fixed domains and scarce capacity, every group inside the exactness
bound of rbgtopo_place_groups_lw."""
from __future__ import annotations

from dataclasses import dataclass
from typing import List

import numpy as np

import groups_gen as gg
import levels_oracle as lo
import lw_oracle as lw
from rbg_b200 import synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, STEP_GANG, Group, GroupsBuilder


@dataclass
class Fleet:
    topo: synth.Topology
    groups: List[Group]
    rp: List[List[tuple]]       # (S, C) per role of every group
    lv: np.ndarray              # [3][n]: level 0 = domain[], level 1 = one domain per node, level 2 = racks of 16
    occ: np.ndarray             # occupancy records (node, gid, level); empty in map mode

    def blob(self) -> np.ndarray:
        return build(self.groups)

    def role_pods(self) -> np.ndarray:
        return np.asarray([sc for g in self.rp for sc in g], dtype=np.int32).reshape(-1, 2)

    def without(self, k: int) -> "Fleet":
        return Fleet(self.topo, self.groups[:k] + self.groups[k + 1:], self.rp[:k] + self.rp[k + 1:], self.lv, self.occ)


def build(groups: List[Group]) -> np.ndarray:
    gb = GroupsBuilder()
    for g in groups:
        gb.add(g)
    return gb.build()


def _fits(g: Group, S: List[int], row_w: int) -> bool:
    """The pod-wave bound of §3.11 item 7 at its worst: need·8 <= 128, every pod and anchor at the largest pair."""
    pods = sum(r[1] * s for r, s in zip(g.roles, S))
    mass = pods + sum(a[2] for a in g.anchors)
    return row_w * (8 * lw.NEED_CAP + max(max(r) for r in g.pair) * mass) < (1 << 24)


def fleet(seed: int, n: int, n_groups: int = 10, scarce: bool = False, levels: bool = False, S_max: int = 8,
          occupancy: bool = False) -> Fleet:
    """levels: co-location levels 1 and 2 as well as 0 and -1 (they need the partitions installed, so the snapshot is
    then in occupancy mode).  occupancy: records of the fleet's own gids and of one outsider on top."""
    rng = np.random.default_rng(seed)
    topo = synth.make_topology(n, seed=seed + 7, tiers=2, owned_frac=0.0 if levels or occupancy else 0.2,
                               max_free=3 if scarce else 8)
    if scarce:
        topo.free = np.where(rng.random(n) < 0.5, 0, topo.free).astype(np.int32)
    if levels or occupancy:
        topo.domain_owner[:] = -1
    lv = np.stack([topo.domain, np.arange(n), np.arange(n) // 16]).astype(np.int32)
    n_dom = len(topo.domain_owner)
    row_w = gg.wsum_max(topo) + 8000
    gids = [int(x) for x in rng.integers(1, 6, size=n_groups)]   # shared gids
    groups, rps = [], []
    for g in range(n_groups):
        q = int(rng.integers(1, 4))
        lvs = np.sort(rng.integers(0, 2, size=q))
        excl = rng.random() < 0.5
        roles = [(int(lvs[i]), int(rng.integers(0, 4)), int(rng.choice([0, 1, 1, 2])),
                  ROLE_EXCLUSIVE if rng.random() < 0.8 else 0) for i in range(q)]
        pair = [[1 if (i == j or rng.random() < 0.5) else 0 for j in range(q)] for i in range(q)]
        anchors = [(int(rng.integers(0, n)), 0, 1)] if rng.random() < 0.3 else []
        fixed = int(rng.integers(0, n_dom)) if excl and rng.random() < 0.25 else -1
        flags = (STEP_EXCLUSIVE if excl else 0) | (STEP_GANG if rng.random() < 0.3 else 0)
        C = [-1, 0, 1, 2] if levels else [-1, 0]
        rp = [(int(rng.integers(1, S_max + 1)), int(rng.choice(C))) for _ in range(q)]
        grp = Group(gid=gids[g], roles=roles, pair=pair, anchors=anchors, flags=flags, fixed_domain=fixed)
        while not _fits(grp, [s for s, _ in rp], row_w):
            k = max(range(q), key=lambda i: grp.roles[i][1] * rp[i][0])
            r = grp.roles[k]
            grp.roles[k] = (r[0], r[1] - 1, r[2], r[3])
        groups.append(grp)
        rps.append(rp)
    occ = np.zeros((0, 3), dtype=np.int32)
    if occupancy:
        occ = lo.random_occ(rng, n, 2, sorted(set(gids))[:3] + [99999], max(1, n // 8))
    return Fleet(topo, groups, rps, lv, occ)


def owner0(f: Fleet) -> np.ndarray:
    """The derived level-0 owner of every node once the fleet's levels and records are installed."""
    return lo.derive_level_owner(f.lv, f.occ)[0]


SEEDS = [(1, 7, False), (2, 31, True), (3, 64, False), (4, 130, True), (5, 257, True), (6, 513, False)]
