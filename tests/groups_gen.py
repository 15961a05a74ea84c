"""Seeded generator of GROUPS blobs at the limits of the ABI (test infrastructure).

The plugin's own fleets (synth shapes) stay far inside what include/rbgtopo.h admits: at most 3 role rows
per wave, 5 roles per group, 0/1 symmetric pair matrices with a unit diagonal, demand 0/1, anchor count 1.
`make_case(seed, n_nodes)` builds a snapshot and a GROUPS blob that reach the limits instead: 16-role
groups, levels of 9+ pending roles (a wave of exactly 8 role rows, the next one starting mid-level),
waves of exactly 32 replicas, roles split across waves, asymmetric pair weights 0-3 with zero diagonals,
all-zero pair rows, demands 0 / 2-4 / above every node's capacity, role-disable-exclusive roles,
preset and self-owned exclusive domains, anchor counts > 1 in repeated records and on full nodes, and
gang / non-gang groups under scarce capacity.  `coverage()` reports which of those a set of cases
reached, so a test can assert that its seeds still reach every one.

Every wave stays under the exactness bound of DESIGN.md §3.4, checked conservatively: every pending
replica of the group is counted as a future anchor (`exact_ok`)."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List

import numpy as np

from rbg_b200 import synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, STEP_GANG, Group, GroupsBuilder

MAX_STEP_ROLES, MAX_STEP_REPLICAS, NEED_CAP, F_CAP, SELF_W = 8, 32, 16, 8, 8000

# The seed set of the GPU parity tests: (seed, nodes, scarce capacity, exclusive groups allowed).  N < 32 gives key lists
# shorter than K, N % 4 != 0 runs the tail mask of the dense-matrix kernel, in its exclusive (<true>) and plain (<false>)
# instantiation.  tests/test_groups_gen.py asserts that together they reach every entry of BULLETS.
CASES = [(1, 7, False, True), (2, 31, True, True), (3, 33, False, True), (4, 130, True, True), (5, 2049, False, True),
         (6, 4097, True, True), (7, 7, False, False), (8, 33, True, False), (9, 2049, False, False), (10, 1, False, True)]


@dataclass
class Case:
    topo: synth.Topology
    groups: List[Group]
    blob: np.ndarray
    wsum_max: int


def wsum_max(topo) -> int:
    cs = np.concatenate([[0], np.cumsum(topo.edge_w, dtype=np.int64)])
    return int((cs[topo.row_ptr[1:]] - cs[topo.row_ptr[:-1]]).max())


def exact_ok(g: Group, row_w: int) -> bool:
    """(max row weight sum + 8000) x (need·8 + Σ pair·(anchors + every pending replica)) < 2^24 for every role."""
    q = len(g.roles)
    mass = [r[1] for r in g.roles]
    for node, role, cnt in g.anchors:
        mass[role] += cnt
    return all((row_w + SELF_W) * (NEED_CAP * F_CAP + sum(g.pair[r][j] * mass[j] for j in range(q))) < (1 << 24)
               for r in range(q))


def waves_of(roles) -> List[List[tuple]]:
    """The wave rule of DESIGN.md §3.2 over a role table [(level, pending, demand, flags)]: (role, first, count)."""
    waves, cur, n, prev = [], [], 0, None
    for ri, (lv, pend, _, _) in enumerate(roles):
        if lv != prev and cur:
            waves.append(cur)
            cur, n = [], 0
        prev = lv
        left, first = pend, 0
        while left > 0:
            if n == MAX_STEP_REPLICAS or len(cur) == MAX_STEP_ROLES:
                waves.append(cur)
                cur, n = [], 0
            take = min(left, MAX_STEP_REPLICAS - n)
            cur.append((ri, first, take))
            n, left, first = n + take, left - take, first + take
    if cur:
        waves.append(cur)
    return waves


def _pair(rng, q: int, zero_row: bool) -> List[List[int]]:
    p = rng.integers(0, 4, size=(q, q))
    np.fill_diagonal(p, 0)
    if zero_row:
        p[int(rng.integers(0, q))] = 0
    return p.tolist()


def _wide(rng, demand_big: int) -> List[tuple]:
    """16 roles: a level of 10 (>= 9 pending, zeros in between), a level with nothing pending, a level whose
    roles sum past 32 (a wave of exactly 32, a role split across two waves)."""
    roles = []
    pend0 = [int(x) for x in rng.integers(1, 4, size=10)]
    pend0[int(rng.integers(2, 9))] = 0                                      # zero-pending role between pending ones
    for i in range(10):
        roles.append([0, pend0[i], int(rng.choice([0, 1, 2, 3, 4])), ROLE_EXCLUSIVE])
    for _ in range(3):
        roles.append([1, 0, 1, ROLE_EXCLUSIVE])                              # nothing pending in level 1
    a = int(rng.integers(17, 26))
    for pend in (a, 32 - a + int(rng.integers(1, 6)), int(rng.integers(0, 4))):
        roles.append([2, pend, int(rng.choice([1, 2])), ROLE_EXCLUSIVE])
    if rng.random() < 0.3:
        roles[int(rng.integers(0, 10))][2] = demand_big                     # never fits any node
    return [tuple(r) for r in roles]


def _small(rng) -> List[tuple]:
    q = int(rng.integers(1, 6))
    lv = np.sort(rng.integers(0, 3, size=q))
    return [(int(lv[i]), int(rng.choice([0, 1, 2, 3, 4, 5, 31, 32, 33])), int(rng.choice([0, 1, 1, 2, 3])), ROLE_EXCLUSIVE)
            for i in range(q)]


def make_case(seed: int, n_nodes: int, n_groups: int = 10, scarce: bool = False, exclusive: bool = True,
              tiers: int = 2) -> Case:
    """exclusive = False: no exclusive group (the dense-matrix kernel's <false> instantiation).  tiers = 2 keeps node
    degrees low enough that every group's table of patched nodes fits k_plan_group's shared memory."""
    rng = np.random.default_rng(seed)
    topo = synth.make_topology(n_nodes, seed=seed + 1, tiers=tiers, owned_frac=0.2 if n_nodes >= 16 else 0.0, max_free=4)
    free = topo.free.copy()
    if scarce:
        free[rng.random(n_nodes) < 0.7] = 0
    topo.free = free.astype(np.int32)
    demand_big = int(free.max()) + 1
    n_dom = len(topo.domain_owner)
    row_w = wsum_max(topo)
    gids = [100 + 7 * g for g in range(n_groups)]
    groups: List[Group] = []
    for g in range(n_groups):
        kind = (g + seed) % 5                      # 0 wide, 1 wide exclusive, 2 small, 3 idle, 4 small exclusive
        if kind in (0, 1):
            roles = _wide(rng, demand_big)
        elif kind == 3:
            roles = [(0, 0, 1, ROLE_EXCLUSIVE), (1, 0, 2, 0)]                 # nothing pending
        else:
            roles = _small(rng)
        excl = (kind in (1, 3, 4) or rng.random() < 0.2) and exclusive
        if excl:                                   # role-disable-exclusive roles, one of them first in its wave
            roles = [(lv, p, d, f if rng.random() < 0.7 else 0) for lv, p, d, f in roles]
            w0 = waves_of(roles)
            if w0:
                wi = int(rng.integers(0, len(w0)))
                r0 = w0[wi][0][0]
                roles[r0] = roles[r0][:3] + (0,)
        q = len(roles)
        pair = _pair(rng, q, zero_row=rng.random() < 0.5)
        anchors = []
        for _ in range(int(rng.integers(0, 5))):
            node, role = int(rng.integers(0, n_nodes)), int(rng.integers(0, q))
            anchors.append((node, role, int(rng.integers(1, 4))))
            if rng.random() < 0.3:
                anchors.append((node, role, int(rng.integers(1, 3))))    # repeated (node, role) record
        full = np.nonzero(topo.free == 0)[0]
        if len(full) and rng.random() < 0.5:
            anchors.append((int(rng.choice(full)), int(rng.integers(0, q)), 2))   # scheduled pod on a full node
        fixed = -1
        if excl and rng.random() < 0.5:
            fixed = int(rng.integers(0, n_dom))
        if excl and rng.random() < 0.6 and n_dom > 1:
            d = fixed if fixed >= 0 else int(rng.integers(0, n_dom))
            topo.domain_owner[d] = gids[g]                                    # a domain the group owns itself
        gang = rng.random() < 0.4
        grp = Group(gid=gids[g], roles=roles, pair=pair, anchors=anchors,
                    flags=(STEP_EXCLUSIVE if excl else 0) | (STEP_GANG if gang else 0), fixed_domain=fixed)
        while not exact_ok(grp, row_w):            # lower the heaviest weight until the bound holds
            p = np.asarray(grp.pair)
            p[np.unravel_index(int(np.argmax(p)), p.shape)] -= 1
            grp.pair = p.tolist()
        groups.append(grp)
    gb = GroupsBuilder()
    for grp in groups:
        gb.add(grp)
    return Case(topo, groups, gb.build(), row_w)


BULLETS = ("q16", "level_ge9", "wave_32", "role_split", "zero_between", "empty_level", "idle_group", "asym_pair",
           "zero_pair_row", "demand_0", "demand_2_4", "demand_big", "opt_out", "opt_out_first_excl", "fixed_domain",
           "self_owned", "anchor_count", "anchor_repeat", "anchor_full", "status1", "status2")


def coverage(case: Case, status=None) -> Dict[str, bool]:
    """Which limits of the ABI the case reaches; `status` = the oracle's per-group status (status 1 / 2 bullets)."""
    c = dict.fromkeys(BULLETS, False)
    free_max = int(case.topo.free.max())
    for g in case.groups:
        q = len(g.roles)
        p = np.asarray(g.pair)
        excl = bool(g.flags & STEP_EXCLUSIVE)
        c["q16"] |= q == 16
        levels: Dict[int, List[int]] = {}
        for ri, r in enumerate(g.roles):
            levels.setdefault(r[0], []).append(ri)
        for ids in levels.values():
            pend = [g.roles[i][1] for i in ids]
            c["level_ge9"] |= sum(x > 0 for x in pend) >= 9
            c["empty_level"] |= sum(pend) == 0
            nz = [i for i, x in enumerate(pend) if x > 0]
            c["zero_between"] |= any(pend[i] == 0 for i in range(nz[0], nz[-1])) if nz else False
        c["idle_group"] |= sum(r[1] for r in g.roles) == 0
        waves = waves_of(g.roles)
        seen = set()
        for w in waves:
            c["wave_32"] |= sum(x[2] for x in w) == 32
            c["role_split"] |= w[0][0] in seen
            seen.update(x[0] for x in w)
            c["opt_out_first_excl"] |= excl and not (g.roles[w[0][0]][3] & ROLE_EXCLUSIVE)
        c["asym_pair"] |= bool((p != p.T).any()) and p.max() >= 2 and not np.diag(p).any()
        c["zero_pair_row"] |= any(not p[r].any() and g.roles[r][1] > 0 for r in range(q))
        for _, pend, dem, fl in g.roles:
            if pend > 0:
                c["demand_0"] |= dem == 0
                c["demand_2_4"] |= 2 <= dem <= 4
                c["demand_big"] |= dem > free_max
                c["opt_out"] |= not (fl & ROLE_EXCLUSIVE)
        c["fixed_domain"] |= excl and g.fixed_domain >= 0
        c["self_owned"] |= excl and bool((case.topo.domain_owner == g.gid).any())
        keys = [(n, r) for n, r, _ in g.anchors]
        c["anchor_count"] |= any(cnt > 1 for _, _, cnt in g.anchors)
        c["anchor_repeat"] |= len(set(keys)) < len(keys)
        c["anchor_full"] |= any(case.topo.free[n] == 0 for n, _, _ in g.anchors)
    if status is not None:
        st = [int(s) for s in status]
        c["status1"] = 1 in st
        c["status2"] = 2 in st
    return c
