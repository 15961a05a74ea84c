"""Seeded cases of exclusive topology at its limits (DESIGN.md §3.9; test infrastructure).

Each builder returns a LevelsCase (snapshot, level partitions, records, and the GROUPS blob or steps it places) and
has a precondition, a function that returns the facts the case exists for; tests/test_oracle_levels_limits.py asserts
them on the CPU and tests/test_gpu_levels_limits.py re-asserts the stride counts from the device's real SM count.

derivation     N = 2^20 + 1, seven levels, ~7.4 M domains and >= 600 000 records: every loop of k_level_owner goes
               past its first grid stride; 100 000 records of 3 000 gids on one level-0 domain, 50 000 of one gid on one
               node, gids 0 and 2^31 - 1, a gid keyed only at level 7, 32 gids on one node;
reinstalls     7 hostname levels, then 2 coarse ones, then 7 with a larger total domain count, then an occupancy-only
               refresh without records and one with records;
keys47         groups_gen fleets with every group at level 4 + g % 4 (fixed domains renumbered into the group's level,
               the last domain of level 7, fixed domain 0 of a single-domain level), scarce capacity, failing gangs;
               inside the domains the groups place in, owner_L and owner_{L-4} differ;
level_split    groups at levels 6 and 7 whose domain holds nodes free at L but blocked at L - 4, and those nodes rank
               first in the group's dense row: a level read with two bits anywhere changes the ranked alternates;
steps47        a step batch at levels 4..7 with a heavy anchored step past k_select_assign_fast's shared memory;
wide47         a 16-role group at level 6 whose table of patched nodes does not fit k_plan_group's shared memory;
ragged         N in {1, 31, 32, 33}, every group at level 7;
hostname_1m    N = 2^20 + 1, hostname-like levels 5 and 7, the only usable node last in the background order;
gid_ends       exclusive groups of gids 0 and 2^31 - 1 at level 6 next to records of both;
ceiling        total domain count exactly 0x3FFFFFF0 on 64 nodes, and one past it.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

import groups_gen as gg
import levels_oracle as lo
import levels_view as lvw
from rbg_b200 import synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, STEP_GANG, Group, GroupsBuilder, Step

H100_SMS = 132                       # SMs of an H100 SXM5
LEVEL_OWNER_CTAS_PER_SM, LEVEL_OWNER_THREADS = 8, 256   # k_level_owner's grid cap (rbgtopo_set_exclusive_levels)
MAX_TOTAL_DOMAINS = 0x3FFFFFF0       # domains of all levels together (RBGTOPO_ELIMIT above)
GID_MAX = (1 << 31) - 1
EMIT_CHUNK = 2048


def grid_strides(work: int, sm_count: int = H100_SMS) -> int:
    """Grid-stride rounds of one k_level_owner loop over `work` items: the grid is min(ceil(work / 256), 8 * SMs)
    CTAs of 256 threads."""
    ctas = max(1, min(-(-work // LEVEL_OWNER_THREADS), sm_count * LEVEL_OWNER_CTAS_PER_SM))
    return -(-work // (ctas * LEVEL_OWNER_THREADS))


@dataclass
class LevelsCase:
    topo: synth.Topology
    lv: np.ndarray                   # [n_levels + 1][n], row 0 = topo.domain
    nd: List[int]                    # domains per level, level 0 first
    occ: np.ndarray                  # (node, gid, level) records
    gblob: Optional[np.ndarray] = None
    steps: List[Step] = field(default_factory=list)
    extra: dict = field(default_factory=dict)

    @property
    def total_domains(self) -> int:
        return int(sum(self.nd))


def build_groups(groups) -> np.ndarray:
    gb = GroupsBuilder()
    for g in groups:
        gb.add(g)
    return gb.build()


def plain_topology(n: int, domain, free: int = 4, tiers: int = 1) -> synth.Topology:
    """NVLink cliques of 8 (tiers = 1: no other links), uniform free, the given level-0 domains, no owners."""
    t = synth.make_topology(n, seed=5, tiers=tiers, max_free=1)
    t.free = np.full(n, free, np.int32)
    t.domain = np.asarray(domain, np.int32)
    t.domain_owner = np.full(int(t.domain.max()) + 1, -1, np.int32)
    return t


def compact(d) -> np.ndarray:
    return np.unique(np.asarray(d, np.int64), return_inverse=True)[1].astype(np.int32)


# ---------------------------------------------------------------- derivation past one grid stride
FULL_N = (1 << 20) + 1


def derivation(n: int = FULL_N, seed: int = 1, n_records: int = 610_000) -> LevelsCase:
    """At N = FULL_N as described above; at a smaller N (for the literal oracle) the same shapes with the special nodes,
    the level-0 domain size and the record counts scaled down with N."""
    rng = np.random.default_rng(seed)
    ids = np.arange(n, dtype=np.int64)

    def at(x):                                  # node x of the full-size case, scaled to this N
        return int(x) * n // FULL_N

    def count(x):
        return max(1, int(x) * n // FULL_N) if n < FULL_N else int(x)
    dsize = 4096 if n == FULL_N else max(16, n // 64)
    bg = at(250_000)                           # the background's nodes: [0, bg)
    topo = plain_topology(n, ids // dsize)
    perm = rng.permutation(n)
    # level 7: a random hash among the background's nodes (collisions), one domain per node elsewhere
    l7 = np.where(ids < bg, rng.integers(0, 2 * bg, n), 2 * bg + ids)
    lv = np.stack([topo.domain, ids, ids // 16, (ids + 128) // 256, np.zeros(n, np.int64), perm, 2 * ids,
                   l7]).astype(np.int32)
    # levels 5..7 declare 2N domains each (most of them empty): the tables phase 0 clears are ~7.3 M domains
    nd = [int(lv[0].max()) + 1, n, int(lv[2].max()) + 1, int(lv[3].max()) + 1, 1, 2 * n, 2 * n, 2 * n]
    parts = []
    # 100 000 records on level-0 domain 5 from 3 000 gids: every node there holds >= 2 distinct gids
    i = np.arange(count(100_000))
    parts.append(np.stack([5 * dsize + i % dsize, 10_000 + i % 3000, np.array([0, 1, 2, 3, 5, 6, 7])[i % 7]], 1))
    # 50 000 records of gid 7 on one node, at every level but the single-domain one
    i = np.arange(count(50_000))
    parts.append(np.stack([np.full(len(i), at(700_000)), np.full(len(i), 7), np.array([0, 1, 2, 3, 5, 6, 7])[i % 7]], 1))
    # the ends of int32, alone on their nodes at the hostname level (17 apart: neighbouring racks of 16)
    ends = ((at(900_000), 0), (at(900_000) + 17, GID_MAX))
    parts.append(np.array([[v, g, 1] for v, g in ends]))
    # gid 555 keyed only at level 7
    k7 = (555, at(300_000), min(100, count(100)))
    parts.append(np.stack([k7[1] + np.arange(k7[2]), np.full(k7[2], 555), np.full(k7[2], 7)], 1))
    # 32 distinct gids on one node
    parts.append(np.stack([np.full(32, at(400_000)), 20_000 + np.arange(32), np.full(32, 1)], 1))
    # background: runs of 64 nodes share a gid, keyed at levels that stay local (never 0, 3 or the single domain)
    k = count(n_records) - sum(len(p) for p in parts)
    node = rng.integers(0, bg, k)
    parts.append(np.stack([node, 100 + (node // 64) % 40, np.array([1, 2, 5, 6, 7])[rng.integers(0, 5, k)]], 1))
    occ = np.concatenate(parts).astype(np.int32)
    occ = occ[rng.permutation(len(occ))]
    return LevelsCase(topo, lv, nd, occ, extra=dict(contention_domain=5, same_gid_node=at(700_000), ends=ends,
                                                   keyed7=k7, crowd_node=at(400_000)))


def derivation_facts(c: LevelsCase, owner: Optional[np.ndarray] = None, sm_count: int = H100_SMS) -> dict:
    """The stride counts, the record shapes, and (given the derived owners) what the records must leave behind."""
    n = c.topo.n
    occ = c.occ.astype(np.int64)
    f = dict(n=n, levels=c.lv.shape[0] - 1, records=len(occ),
             phase0=grid_strides(2 * c.total_domains, sm_count), phase1=grid_strides(len(occ), sm_count),
             phase2=grid_strides(n, sm_count), ragged=n % 32 != 0 and n % EMIT_CHUNK != 0)
    cd = c.extra["contention_domain"]
    m = c.lv[0][occ[:, 0]] == cd
    f["contention_records"] = int(m.sum())
    f["contention_gids"] = len(np.unique(occ[m, 1]))
    f["same_gid_records"] = int(((occ[:, 0] == c.extra["same_gid_node"]) & (occ[:, 1] == 7)).sum())
    f["gids_at_ends"] = {0, GID_MAX} <= set(occ[:, 1].tolist())
    g7, n0, cnt = c.extra["keyed7"]
    f["keyed7_only_at_7"] = set(occ[occ[:, 1] == g7, 2].tolist()) == {7}
    f["crowd_gids"] = len(np.unique(occ[occ[:, 0] == c.extra["crowd_node"], 1]))
    if owner is not None:
        nodes = np.flatnonzero(c.lv[0] == cd)
        # every level that holds a contention record: -2 at each of its domains' nodes
        f["contention_blocked"] = all((owner[L, nodes] == lo.BLOCKED).all() for L in range(owner.shape[0]))
        f["same_gid_kept"] = int(owner[1, c.extra["same_gid_node"]]) == 7
        f["ends_kept"] = all(int(owner[1, v]) == g for v, g in c.extra["ends"])
        span = slice(n0, n0 + cnt)
        f["keyed7_everywhere"] = all(((owner[L, span] == g7) | (owner[L, span] == lo.BLOCKED)).all()
                                     for L in range(owner.shape[0])) and bool((owner[1, span] == g7).all())
        f["crowd_blocked"] = int(owner[1, c.extra["crowd_node"]]) == lo.BLOCKED
        f["kinds"] = {int(x) for x in np.unique(np.clip(owner, -2, 0))}   # {-2, -1, 0}: blocked, free, owned
    return f


# ---------------------------------------------------------------- partition reinstalls
def reinstalls(n: int = 4097, seed: int = 2):
    """[(level rows 1.. or None, records, nd of levels 1..)] to install in order, on one snapshot."""
    rng = np.random.default_rng(seed)
    topo = plain_topology(n, np.arange(n) // 512, tiers=2)
    ids = np.arange(n)

    def recs(k, n_levels, gids):
        lvls = rng.integers(1, n_levels + 1, k)
        return np.stack([rng.integers(0, n, k), rng.choice(gids, k), lvls], 1).astype(np.int32)

    host7 = np.stack([rng.permutation(n) for _ in range(7)]).astype(np.int32)
    coarse2 = np.stack([ids // 300, ids // 1000]).astype(np.int32)
    big7 = np.stack([compact(rng.integers(0, n // (L + 1) + 1, n)) for L in range(7)])
    nd_big = [3 * n] * 7
    seq = [(host7, recs(n // 3, 7, [3, 5, 8, 13]), [n] * 7),
           (coarse2, recs(n // 5, 2, [3, 21]), [int(r.max()) + 1 for r in coarse2]),
           (big7, recs(n // 4, 7, [3, 5, 34]), nd_big),
           (None, np.zeros((0, 3), np.int32), None),
           (None, recs(n // 6, 7, [55, 89]), None)]
    return topo, seq


# ---------------------------------------------------------------- keys 4..7 on every path
def partitions47(topo, seed: int, kind: str):
    """Levels 1..7.  'single': level 6 is one domain (records then carry one gid); 'random': nested and non-nested
    random partitions, hostname-like levels 1 and 4."""
    n = topo.n
    rng = np.random.default_rng(seed)
    nested = lo.random_levels(rng, n, topo.domain, 3, [True, False, True])
    rows = [topo.domain, np.arange(n), nested[1], nested[2], rng.permutation(n), nested[3]]
    rows.append(np.zeros(n, np.int64) if kind == "single" else compact(rng.integers(0, max(2, n // 50), n)))
    rows.append(compact(nested[1].astype(np.int64) * 3 + rng.integers(0, 3, n)))
    lv = np.stack(rows).astype(np.int32)
    nd = [len(topo.domain_owner)] + [int(lv[L].max()) + 1 for L in range(1, 8)]
    return lv, nd


def keyed_records(rng, n: int, gids, count: int, levels) -> np.ndarray:
    return np.stack([rng.integers(0, n, count), rng.choice(gids, count), rng.choice(levels, count)], 1).astype(np.int32)


def keys47(seed: int, n: int, kind: str, scarce: bool) -> LevelsCase:
    case = gg.make_case(seed, n, scarce=scarce, exclusive=True)
    topo = case.topo
    lv, nd = partitions47(topo, seed, kind)
    rng = np.random.default_rng(seed + 77)
    ng = int(case.blob[2])
    levels = [4 + g % 4 for g in range(ng)]
    gb = lvw.with_levels(case.blob, levels)
    for g in range(ng):
        off = 8 + 12 * g + 2
        if gb[off] >= 0:
            gb[off] = int(rng.integers(0, nd[levels[g]]))          # a fixed domain of the group's own level
    gb[8 + 12 * 3 + 2] = nd[7] - 1                                  # the last domain of level 7 (group 3)
    gb[8 + 12 * 3 + 1] |= STEP_EXCLUSIVE
    gb[8 + 12 * 2 + 2] = 0                                          # fixed domain 0 of level 6 (group 2)
    gb[8 + 12 * 2 + 1] |= STEP_EXCLUSIVE
    gids = [int(gb[8 + 12 * g]) for g in range(ng)]
    r2 = np.random.default_rng(seed + 5)
    if kind == "single":      # one gid owns the single-domain level 6: group 2 places, group 6 finds nothing.  None
        # of its records is keyed at level 6 (that term would reach every node at every level and make all levels
        # look alike) or at level 0
        occ = keyed_records(r2, n, [gids[2]], max(1, n // 20), [1, 2, 3, 4, 5, 7])
    else:                     # never keyed at level 0 or 2 (nested coarse partitions would block most nodes)
        occ = keyed_records(r2, n, gids[:4] + [999], max(1, n // 30), [1, 3, 4, 5, 6, 7])
    return LevelsCase(topo, lv, nd, occ, gblob=gb)


KEYS47 = [(141, 2049, "single", True), (142, 2049, "random", False), (147, 4097, "random", True),
          (144, 4097, "single", False)]


def nests(fine, coarse) -> bool:
    """Every domain of `fine` lies inside one domain of `coarse`."""
    pairs = np.unique(np.asarray(fine, np.int64) << 32 | np.asarray(coarse, np.int64))
    return len(pairs) == len(np.unique(fine))


def split_nodes(c: LevelsCase, owner: np.ndarray, gid: int, level: int, domain: int) -> int:
    """Nodes of `domain` at `level` whose feasibility for `gid` differs between owner_level and owner_{level - 4}:
    what a level read with two bits would get wrong there."""
    inside = c.lv[level] == domain
    ok = [(owner[L] == lo.FREE) | (owner[L] == gid) for L in (level, level - 4)]
    return int((inside & (ok[0] != ok[1])).sum())


def keys47_facts(c: LevelsCase, exp=None, owner=None) -> dict:
    gb = c.gblob
    ng = int(gb[2])
    lvls = [int(gb[8 + 12 * g + 10]) for g in range(ng)]
    fixed = [int(gb[8 + 12 * g + 2]) for g in range(ng)]
    f = dict(levels=set(lvls), last_domain_l7=any(L == 7 and d == c.nd[7] - 1 for L, d in zip(lvls, fixed)),
             fixed_in_level=all(d < c.nd[L] for L, d in zip(lvls, fixed)), single_domain=c.nd[6] == 1,
             nested=nests(c.lv[2], c.lv[0]) and nests(c.lv[7], c.lv[2]), non_nested=not nests(c.lv[3], c.lv[0]))
    f["fixed_0_single"] = any(L == 6 and d == 0 for L, d in zip(lvls, fixed)) and c.nd[6] == 1
    if exp is not None:
        st = [e[1] for e in exp]
        gang = [bool(gb[8 + 12 * g + 1] & STEP_GANG) for g in range(ng)]
        f["status1_at_47"] = sorted({lvls[g] for g in range(ng) if st[g] == 1})
        f["gang_failed"] = any(st[g] == 2 and gang[g] for g in range(ng))
    if exp is not None and owner is not None:
        excl = [bool(gb[8 + 12 * g + 1] & STEP_EXCLUSIVE) for g in range(ng)]
        f["split_in_placed_domains"] = sum(split_nodes(c, owner, int(gb[8 + 12 * g]), lvls[g], exp[g][2])
                                           for g in range(ng) if excl[g] and exp[g][2] >= 0)
    return f


def steps47(c: LevelsCase, seed: int) -> List[Step]:
    """Steps at levels 4..7 (fixed domains of their level on every third), then one heavy step whose anchors'
    closed neighbourhoods put the batch past k_select_assign_fast's shared memory."""
    topo, lv = c.topo, c.lv
    rng = np.random.default_rng(seed)
    gids = [int(c.gblob[8 + 12 * g]) for g in range(int(c.gblob[2]))]
    steps = []
    for k, g in enumerate(gids):
        L = 4 + k % 4
        fixed = -1 if k % 3 else int(lv[L, int(rng.integers(0, topo.n))])
        steps.append(Step(gid=g, roles=[(3, 1, 2, ROLE_EXCLUSIVE), (2, 1, 1, 0)], pair=[[1, 1], [0, 1]],
                          anchors=[(int(rng.integers(0, topo.n)), 0, 1)], flags=STEP_EXCLUSIVE, fixed_domain=fixed,
                          level=L))
    heavy = rng.choice(topo.n, size=min(topo.n, 1500), replace=False)
    steps.append(Step(gid=gids[0], roles=[(2, 1, 1, ROLE_EXCLUSIVE)], pair=[[0]],
                      anchors=[(int(x), 0, 1) for x in heavy], flags=STEP_EXCLUSIVE, level=7))
    return steps


def wide47(seed: int = 7, n: int = 4097, n_anchor_nodes: int = 2000) -> LevelsCase:
    """test_gpu_groups_limits' per-wave fleet at levels 4..7: a 16-role group at level 6 among one-role groups."""
    rng = np.random.default_rng(seed)
    topo = synth.make_topology(n, seed=3, tiers=4, max_free=4)
    p = rng.integers(0, 4, size=(16, 16))
    np.fill_diagonal(p, 0)
    p[:, 15] = 0
    nodes = rng.choice(n, size=n_anchor_nodes, replace=False)
    wide = Group(gid=5, roles=[(0, int(rng.integers(1, 4)), int(rng.integers(0, 3)), ROLE_EXCLUSIVE) for _ in range(16)],
                 pair=p.tolist(), flags=STEP_EXCLUSIVE, level=6,
                 anchors=[(int(x), 15, 1) for x in nodes] + [(int(x), int(rng.integers(0, 15)), 2) for x in nodes[:12]])
    groups = []
    for g in range(20):
        anchors = [(int(rng.integers(0, n)), 0, int(rng.integers(1, 3)))] if g % 3 == 0 else []
        groups.append(Group(gid=10 + g, roles=[(0, int(rng.integers(1, 6)), int(rng.integers(0, 3)), ROLE_EXCLUSIVE)],
                            pair=[[int(rng.integers(0, 4))]], anchors=anchors,
                            flags=STEP_EXCLUSIVE if g % 2 else 0, level=4 + g % 4))
    groups.insert(3, wide)
    lv, nd = partitions47(topo, seed, "random")
    occ = keyed_records(np.random.default_rng(seed + 1), n, [5, 10, 11, 999], n // 10, [1, 3, 4, 5, 6, 7])
    return LevelsCase(topo, lv, nd, occ, gblob=build_groups(groups), extra=dict(wide=wide))


# ---------------------------------------------------------------- nodes free at L, blocked at L - 4
def level_split(n: int = 256) -> LevelsCase:
    """Level 6 = blocks of 32, level 2 = blocks of 32 shifted by 16; level 7 = blocks of 16, level 3 = blocks of 16
    shifted by 8.  A record of gid 60 on node 40 blocks level-2 domain [16, 48) but only level-6 domain [32, 64); one
    of gid 61 on node 150 blocks level-3 domain [136, 152) but only level-7 domain [144, 160).  The cliques [16, 24)
    and [136, 144) have free 4 (every other node 2), so they lead every dense row of the groups placed beside them:
      50  level 6, fixed domain 0 = [0, 32)      — its best nodes 16..23 are free at 6, blocked at 2;
      51  level 7, fixed domain 8 = [128, 144)   — its best nodes 136..143 are free at 7, blocked at 3;
      52  level 6, no fixed domain               — D* = 0, the same nodes as group 50;
      53  level 7, no fixed domain, a replica of demand 3 — lands in [16, 24), which level 3 leaves free."""
    ids = np.arange(n, dtype=np.int64)
    topo = plain_topology(n, ids // 64, free=2)
    topo.free[16:24] = 4
    topo.free[136:144] = 4
    lv = np.stack([topo.domain, ids, (ids + 16) // 32, (ids + 8) // 16, ids // 8, ids, ids // 32,
                   ids // 16]).astype(np.int32)
    nd = [int(r.max()) + 1 for r in lv]
    occ = np.array([[40, 60, 1], [150, 61, 1]], np.int32)
    groups = [Group(gid=50, roles=[(0, 3, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE, level=6,
                    fixed_domain=0),
              Group(gid=51, roles=[(0, 4, 1, ROLE_EXCLUSIVE), (1, 2, 1, 0)], pair=[[1, 0], [1, 1]],
                    flags=STEP_EXCLUSIVE, level=7, fixed_domain=8),
              Group(gid=52, roles=[(0, 2, 2, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE, level=6),
              Group(gid=53, roles=[(0, 1, 3, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE, level=7)]
    return LevelsCase(topo, lv, nd, occ, gblob=build_groups(groups))


# ---------------------------------------------------------------- ragged N at level 7
RAGGED = [1, 31, 32, 33]


def ragged(n: int, seed: int = 150) -> LevelsCase:
    case = gg.make_case(seed + n, n, scarce=n % 2 == 1, exclusive=True)
    topo = case.topo
    rng = np.random.default_rng(seed + n)
    rows = [topo.domain] + [compact(rng.integers(0, max(1, n // k) + 1, n)) for k in (1, 2, 3, 4, 5, 6)]
    rows.append(np.arange(n)[::-1])                                 # level 7 hostname-like
    lv = np.stack(rows).astype(np.int32)
    nd = [len(topo.domain_owner)] + [int(lv[L].max()) + 1 for L in range(1, 8)]
    ng = int(case.blob[2])
    gb = lvw.with_levels(case.blob, [7] * ng)
    for g in range(ng):
        if gb[8 + 12 * g + 2] >= 0:
            gb[8 + 12 * g + 2] = int(rng.integers(0, nd[7]))
    gids = [int(gb[8 + 12 * g]) for g in range(ng)]
    occ = keyed_records(rng, n, gids[:3] + [999], max(1, n // 4), [1, 5, 7])
    return LevelsCase(topo, lv, nd, occ, gblob=gb)


# ---------------------------------------------------------------- hostname keys at a million nodes
def hostname_1m(n: int = (1 << 20) + 1, seed: int = 3) -> LevelsCase:
    """Cliques of 8 with uniform free 3: node n - 1 sits alone in the last clique, so it has the lowest base and the
    highest id, last in the background order.  Levels 5 and 7 are hostname-like; every other node carries a record of
    another gid keyed at level 5.  Groups: 40 (level 5, free choice, 3 replicas), 41 (level 7, fixed to the last
    node's domain, 32 replicas of demand 0), 42 (level 5, same fixed node, 8 replicas of demand 1, not gang),
    43 (level 7, the same as 42 but gang)."""
    rng = np.random.default_rng(seed)
    ids = np.arange(n, dtype=np.int64)
    topo = plain_topology(n, ids // 8192, free=3)
    v = n - 1
    lv = np.stack([topo.domain, ids // 16, ids // 4096, ids // 256, np.zeros(n, np.int64), rng.permutation(n),
                   ids // 2, (n - 1) - ids]).astype(np.int32)
    nd = [int(lv[L].max()) + 1 for L in range(8)]
    others = ids[:-1]
    occ = np.stack([others, 1000 + others % 7, np.full(n - 1, 5)], 1).astype(np.int32)
    d5, d7 = int(lv[5, v]), int(lv[7, v])
    groups = [Group(gid=40, roles=[(0, 3, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE, level=5),
              Group(gid=41, roles=[(0, 32, 0, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE, level=7,
                    fixed_domain=d7),
              Group(gid=42, roles=[(0, 8, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE, level=5,
                    fixed_domain=d5),
              Group(gid=43, roles=[(0, 8, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE | STEP_GANG,
                    level=7, fixed_domain=d7)]
    return LevelsCase(topo, lv, nd, occ, gblob=build_groups(groups), extra=dict(last=v))


def hostname_facts(c: LevelsCase, owner: Optional[np.ndarray] = None) -> dict:
    n, v = c.topo.n, c.extra["last"]
    deg = np.diff(c.topo.row_ptr)
    f = dict(n=n, hostname_5=c.nd[5] == n, hostname_7=c.nd[7] == n, last_alone=int(deg[v]) == 0 and v == n - 1,
             others_deg=int(deg[:-1].min()), uniform_free=bool((c.topo.free == c.topo.free[0]).all()))
    if owner is not None:
        f["only_usable_5"] = np.flatnonzero(owner[5] == lo.FREE).tolist() == [v]
        f["only_usable_7"] = np.flatnonzero(owner[7] == lo.FREE).tolist() == [v]
    return f


# ---------------------------------------------------------------- gids at the ends of int32
def gid_ends(n: int = 2049, seed: int = 4) -> LevelsCase:
    rng = np.random.default_rng(seed)
    topo = synth.make_topology(n, seed=seed, tiers=2, max_free=4)
    topo.domain_owner[:] = -1
    lv, nd = partitions47(topo, seed, "random")
    occ = keyed_records(rng, n, [0, GID_MAX], n // 12, [1, 5, 6, 7])
    groups = [Group(gid=0, roles=[(0, 5, 1, ROLE_EXCLUSIVE), (1, 3, 1, 0)], pair=[[1, 1], [1, 1]],
                    flags=STEP_EXCLUSIVE, level=6),
              Group(gid=GID_MAX, roles=[(0, 6, 1, ROLE_EXCLUSIVE)], pair=[[2]], flags=STEP_EXCLUSIVE, level=6),
              Group(gid=GID_MAX, roles=[(0, 4, 2, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE, level=6,
                    fixed_domain=int(lv[6][int(occ[0, 0])])),
              Group(gid=7, roles=[(0, 4, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE, level=6)]
    return LevelsCase(topo, lv, nd, occ, gblob=build_groups(groups))


# ---------------------------------------------------------------- the domain ceiling
def ceiling(n: int = 64, over: int = 0) -> LevelsCase:
    """One level above 0 whose declared count brings the total to MAX_TOTAL_DOMAINS + over; node 0 sits in its last
    domain, the others in a few low ones."""
    topo = plain_topology(n, np.arange(n) // 16, tiers=2)
    nd1 = MAX_TOTAL_DOMAINS + over - len(topo.domain_owner)
    l1 = np.arange(n, dtype=np.int64) % 5
    l1[0] = nd1 - 1
    lv = np.stack([topo.domain, l1]).astype(np.int32)
    occ = np.array([[0, 9, 1], [1, 9, 0], [2, 11, 1], [7, 11, 1], [7, 9, 1], [20, GID_MAX, 0]], np.int32)
    g = Group(gid=9, roles=[(0, 4, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE, level=1, fixed_domain=nd1 - 1)
    return LevelsCase(topo, lv, [len(topo.domain_owner), nd1], occ, gblob=build_groups([g]))
