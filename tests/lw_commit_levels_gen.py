"""Committed leader-worker batches at exclusive levels (DESIGN.md §3.16; test infrastructure): lw_commit_gen's groups
and (S, C) at exclusive levels 0..3 of commit_levels_gen's partitions, co-location levels over the same partitions,
records of the batch's gids and of one gid outside it at every level, the oracle's expected results and the
brute-force anti-affinity check of placed pods (levels_oracle.violates)."""
from __future__ import annotations

import dataclasses
from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np

import levels_oracle as lo
import lw_commit_gen as lg
import lw_committed_oracle as lco
import lw_oracle as lw
from commit_levels_gen import KEYS, partitions
from committed_levels_oracle import group_levels
from lw_committed_levels_oracle import run_lw_committed_levels, run_lw_committed_levels_ranked
from rbg_b200 import synth
from rbg_b200.blob import Group


@dataclass
class LvFleet:
    topo: synth.Topology
    groups: List[Group]
    rp: List[List[tuple]]
    lv: np.ndarray          # [4][n], row 0 = the snapshot's domain
    nd: List[int]
    occ: np.ndarray         # (node, gid, level) records

    def blob(self) -> np.ndarray:
        return lg.build(self.groups)

    def role_pods(self) -> np.ndarray:
        return np.asarray([sc for g in self.rp for sc in g], dtype=np.int32).reshape(-1, 2)

    def owner(self) -> np.ndarray:
        return lo.derive_level_owner(self.lv, self.occ)

    def sub(self, keep: Sequence[int]) -> "LvFleet":
        return LvFleet(self.topo, [self.groups[k] for k in keep], [self.rp[k] for k in keep], self.lv, self.nd, self.occ)

    def expected(self, **kw):
        return run_lw_committed_levels(self.topo, self.blob(), self.role_pods(), self.lv, self.owner(), self.nd, **kw)

    def expected_ranked(self, n_alt: int):
        return run_lw_committed_levels_ranked(self.topo, self.blob(), self.role_pods(), n_alt, self.lv, self.owner(),
                                              self.nd)


def fleet(seed: int, n: int, n_groups: int = 10, scarce: bool = False, kind: str = "mixed",
          levels: Optional[Sequence[int]] = None, S_max: int = 8) -> LvFleet:
    """Group g at exclusive level levels[g] (default: drawn from 0..3); fixed domains of levels >= 1 redrawn in that
    level; C drawn from -1..3."""
    f = lg.fleet(seed, n, n_groups=n_groups, scarce=scarce, levels=True, S_max=S_max)
    rng = np.random.default_rng(seed + 91)
    lv, nd = partitions(f.topo, seed, kind)
    levels = [int(x) for x in rng.integers(0, 4, size=n_groups)] if levels is None else list(levels)
    groups, rps = [], []
    for g, L in zip(f.groups, levels):
        fixed = g.fixed_domain
        if fixed >= 0 and L > 0:
            fixed = int(rng.integers(0, nd[L]))
        groups.append(dataclasses.replace(g, level=L, fixed_domain=fixed))
    for rp in f.rp:
        rps.append([(S, int(rng.choice([-1, 0, 1, 2, 3]))) for S, _ in rp])
    gids = sorted({g.gid for g in groups})
    occ = lo.random_occ(np.random.default_rng(seed + 5), n, 3, gids[:4] + [999], max(1, n // 8))
    return LvFleet(f.topo, groups, rps, lv, nd, occ)


def violations(lv, occ, gblob, role_pods, assign, status) -> list:
    """Placed participating pods of exclusive groups that break a required anti-affinity term of the records or of an
    earlier group's placed participating pods (levels_oracle.violates checks both directions)."""
    G = lco.groups_of(gblob, role_pods)
    levels = group_levels(gblob)
    pods = [tuple(int(x) for x in r) for r in np.asarray(occ).reshape(-1, 3)]
    bad = []
    for g, X in enumerate(G):
        if not (X.flags & lw.STEP_EXCLUSIVE):
            continue
        mine = []
        for ri in range(X.q):
            if not X.rflags[ri] & lw.ROLE_EXCLUSIVE:
                continue
            lo_ = X.pod0 + X.first_pod[ri]
            for node in assign[lo_:lo_ + X.pending[ri] * X.S[ri]]:
                if node < 0:
                    continue
                if lo.violates(lv, KEYS[:len(lv)], np.array(pods, dtype=np.int64).reshape(-1, 3), X.gid, levels[g],
                               int(node)):
                    bad.append((g, ri, int(node)))
                mine.append((int(node), X.gid, levels[g]))
        if int(status[g]) != 2:
            pods += mine
    return bad


# (seed, n, scarce, kind): N = 1 .. 4 097, ragged N, the three partition kinds
SEEDS = [(1, 1, False, "mixed"), (2, 33, True, "random"), (3, 64, False, "edge"), (4, 130, True, "mixed"),
         (5, 257, True, "random"), (6, 513, False, "edge"), (7, 2049, True, "mixed"), (8, 4097, False, "random")]
