"""Committed batches at exclusive levels (DESIGN.md §3.8 / §3.9; test infrastructure): commit_gen-style batches whose
groups sit at levels 0..3 of the 'mixed' / 'random' / 'edge' partitions of test_gpu_levels_place.py, with records of
the batch's gids and of one gid outside it, the expected results of
committed_levels_oracle.run_fleet_committed_levels, and the brute-force check of the results against the reference's anti-affinity terms (levels_oracle.violates)."""
from __future__ import annotations

from dataclasses import dataclass
from typing import List

import numpy as np

import commit_gen as cg
import levels_oracle as lo
from committed_levels_oracle import group_levels, run_fleet_committed_levels
from committed_oracle import result_arrays
from oracle import wave_loop
from rbg_b200 import synth

KEYS = [f"example.com/level-{L}" for L in range(8)]


def partitions(topo, seed, kind):
    from test_gpu_levels_place import partitions as p
    return p(topo, seed, kind)


@dataclass
class LevelCase:
    name: str
    topo: synth.Topology
    lv: np.ndarray          # [n_levels + 1][n], row 0 = the snapshot's domain
    nd: List[int]           # domain count per level
    blob: np.ndarray
    occ: np.ndarray         # (node, gid, level) records


def with_levels(case: cg.Case, seed: int, kind: str, fixed_level: bool = True, levels=None) -> LevelCase:
    """The batch of a commit_gen case with group g at level levels[g] (default g % 4), fixed domains of levels >= 1
    redrawn in the group's level (or dropped), and records at levels 0..3."""
    topo = case.topo
    topo.domain_owner[:] = -1     # occupancy mode: the records decide every owner
    lv, nd = partitions(topo, seed, kind)
    rng = np.random.default_rng(seed + 77)
    ng = int(case.blob[2])
    levels = [g % 4 for g in range(ng)] if levels is None else list(levels)
    gb = np.array(case.blob, dtype=np.int32, copy=True)
    for g in range(ng):
        gb[8 + 12 * g + 10] = levels[g]
        off = 8 + 12 * g + 2
        if gb[off] >= 0 and levels[g] > 0:
            gb[off] = int(rng.integers(0, nd[levels[g]])) if fixed_level else -1
    gids = sorted({int(gb[8 + 12 * g]) for g in range(ng)})
    occ = lo.random_occ(np.random.default_rng(seed + 5), topo.n, 3, gids[:4] + [999], max(1, topo.n // 8))
    return LevelCase(f"{case.name}@{kind}", topo, lv, nd, gb, occ)


def cases() -> List[LevelCase]:
    """N in {1, 33, 130, 2049, 4097} on the three partition kinds, scarce and domain-racing batches, with and
    without fixed domains at levels >= 1."""
    out = [with_levels(cg.scarce(200, 1, n_groups=6, exclusive=0.8), 200, "mixed")]
    for i, (n, kind) in enumerate([(33, "mixed"), (33, "random"), (130, "random"), (130, "edge"), (2049, "mixed"),
                                   (2049, "edge"), (4097, "random"), (4097, "edge")]):
        out.append(with_levels(cg.domains(210 + i, n), 210 + i, kind, fixed_level=i % 2 == 0))
        out.append(with_levels(cg.scarce(230 + i, n, n_groups=20, exclusive=0.7), 230 + i, kind,
                               fixed_level=i % 2 == 1))
    return out


def expected(c: LevelCase, fast: bool = True):
    owner = lo.derive_level_owner(c.lv, c.occ)
    states = run_fleet_committed_levels(c.topo, wave_loop.groups_from_blob(c.blob), group_levels(c.blob), c.lv, owner,
                                        c.nd, fast=fast)
    return result_arrays(states)


def violations(lv, occ, gblob, assign, status) -> list:
    """Placed participating replicas of exclusive groups that break a required anti-affinity term of the records or of
    an earlier group's placed participating pods (levels_oracle.violates, both directions)."""
    groups = wave_loop.groups_from_blob(gblob)
    levels = group_levels(gblob)
    pods = [tuple(int(x) for x in r) for r in np.asarray(occ).reshape(-1, 3)]
    bad, off = [], 0
    for gi, g in enumerate(groups):
        s = wave_loop.GroupState(g)
        mine = []
        for ri in s.order:
            for _ in range(s.pending[ri]):
                node = int(assign[off])
                off += 1
                if g.exclusive and g.roles[ri].exclusive and node >= 0:
                    if lo.violates(lv, KEYS[:len(lv)], np.array(pods, dtype=np.int64).reshape(-1, 3), g.gid,
                                   levels[gi], node):
                        bad.append((gi, ri, node))
                    mine.append((node, g.gid, levels[gi]))
        if int(status[gi]) != 2:
            pods += mine
    return bad
