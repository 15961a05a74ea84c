"""Seeded committed batches at exclusive levels at their limits (DESIGN.md §3.8 / §3.9; test infrastructure), for the
<true> instantiations of k_plan_group_commit / k_commit_claims / k_commit_diff and commit_owner / commit_note_read.

Every builder returns a Case (snapshot, level partitions, records, GROUPS blob) and the facts its preconditions check;
tests/test_oracle_committed_levels_limits.py asserts them on the oracle alone, tests/test_gpu_committed_levels_limits.py
places the cases on the device.

chain          G one-replica exclusive groups of distinct gids; group i is anchored on its own hub h_i whose two
               neighbours a_i (preferred) and b_i are the only nodes it wants.  Group i takes b_i exactly when group
               i - 1 holds a_{i-1} and that claim reaches a_i: the placements alternate a, b, a, ... and the call takes
               exactly G rounds (group i - 1 settles in round i).  The claim reaches a_i through
                 'P'   the pod term only: a_{i-1} and a_i share a domain at group i's level, not at group i - 1's;
                 'K'   the domain term only, across levels: group i - 1 reports a domain of its level that holds a_i,
                       and a_{i-1} is alone at group i's level;
                 'mix' levels i % 8 (lmask = 0xFF), P links into even i and K links into odd i.
sparse         scarce batches (gangs that fail once earlier claims appear) whose exclusive groups sit at levels {3, 7} or {0, 2, 5} only, their
               non-exclusive groups at the other levels >= 1: lmask's ranks differ from the levels.
offsets        for every adjacent pair of installed levels (L, L + 1), one gid claims domain nd_L - 1 at L and another
               domain 0 at L + 1, by reporting it or as an idle exclusive group (a claim before round 0); later
               groups of other gids are anchored on nodes of both domains.
pods           2 112 participating pods of hostname-level groups (32-replica and 16-role ones) in one zone, read by
               the zone-level groups after them.
gids           gids 0 and 2^31 - 1, one gid at two levels, two gids reporting one domain (only the last reporter
               keeps a later group of the first gid out), records that leave domains blocked (-2) next to claims.
level0         commit_gen's level-0 batches with only their non-exclusive groups moved to levels >= 1: the <true>
               path, lmask within {0}, and the results of the unmoved batch.
"""
from __future__ import annotations

import copy
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import numpy as np

import commit_gen as cg
import levels_limits_cases as llc
import levels_oracle as lo
import levels_view
from committed_levels_oracle import (group_levels, level_owner, participating_pods, run_fleet_committed_levels)
from committed_oracle import group_claims, result_arrays, run_group
from oracle import wave_loop
from rbg_b200 import synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, STEP_GANG, Group

GID_MAX = (1 << 31) - 1


@dataclass
class Case:
    name: str
    topo: synth.Topology
    lv: np.ndarray          # [n_levels + 1][n], row 0 = topo.domain
    nd: List[int]           # domains per level, level 0 first
    occ: np.ndarray         # (node, gid, level) records
    blob: np.ndarray
    rounds: Optional[int] = None
    tags: set = field(default_factory=set)
    extra: dict = field(default_factory=dict)


def _blob(groups) -> np.ndarray:
    gb = cg.build(groups)
    for g, grp in enumerate(groups):
        gb[8 + 12 * g + 10] = grp.level
    return gb


def owner(c: Case) -> np.ndarray:
    return lo.derive_level_owner_fast(c.lv, c.occ) if c.topo.n > 50_000 else lo.derive_level_owner(c.lv, c.occ)


def states(c: Case, **kw):
    return run_fleet_committed_levels(c.topo, wave_loop.groups_from_blob(c.blob), group_levels(c.blob), c.lv,
                                      owner(c), c.nd, fast=True, **kw)


def expected(c: Case, **kw):
    return result_arrays(states(c, **kw))


def lmask(blob) -> int:
    m = 0
    for g in range(int(blob[2])):
        if blob[8 + 12 * g + 1] & STEP_EXCLUSIVE:
            m |= 1 << int(blob[8 + 12 * g + 10])
    return m


def uses_levels(blob) -> bool:
    return any(int(blob[8 + 12 * g + 10]) > 0 for g in range(int(blob[2])))


# ---------------------------------------------------------------- the round machinery, replayed on the oracle
def place_one(c: Case, g: int, earlier, groups, own) -> wave_loop.GroupState:
    """Group g placed seeing the given states of groups 0 .. g - 1 (run_fleet_committed_levels' loop body)."""
    levels = group_levels(c.blob)
    last = [np.full(int(k), lo.FREE, np.int32) for k in c.nd]
    pods, claimed = [], {}
    for s, L in zip(earlier, levels):
        for node, amt in group_claims(s).items():
            claimed[node] = claimed.get(node, 0) + amt
        res = s.result()
        if s.g.exclusive and res["status"] != 2:
            if res["domain"] >= 0:
                last[L][res["domain"]] = s.g.gid
            pods += [(s.g.gid, L, m) for m in participating_pods(s)]
    grp, L = groups[g], levels[g]
    ow = np.array(own, dtype=np.int32, copy=True)
    ow[L] = level_owner(c.lv, own, c.nd, L, last, pods)
    t = levels_view.level_view(c.topo, c.lv, ow, c.nd, L, grp.gid, lo.unused_gid({x.gid for x in groups}))
    gv = copy.copy(grp)
    gv.fixed_domain = 2 * grp.fixed_domain if grp.fixed_domain >= 0 else grp.fixed_domain
    s = run_group(t, gv, claimed, 1, True)
    s.g = grp
    if s.fixed_domain >= 0:
        s.fixed_domain //= 2
    return s


def _key(s) -> tuple:
    r = s.result()
    return tuple(s.assign_in_group_order()), r["status"], r["domain"]


def replay_rounds(c: Case):
    """(rounds, states of every round): round 1 places every group against the snapshot, round r re-runs the groups
    above the lowest group whose result changed in round r - 1 (every changed claim counted as read: the device's
    marks may only over-report), each seeing the earlier groups' results of round r - 1.  Stops at the first round
    whose changes no later group can see."""
    groups = wave_loop.groups_from_blob(c.blob)
    own = owner(c)
    ng = len(groups)
    cur = [place_one(c, g, [], groups, own) for g in range(ng)]
    hist = [cur]
    changed = list(range(ng))
    rounds = 1
    while changed and min(changed) < ng - 1:
        lo_g = min(changed)
        prev = cur
        cur = prev[:lo_g + 1] + [place_one(c, g, prev[:g], groups, own) for g in range(lo_g + 1, ng)]
        changed = [g for g in range(lo_g + 1, ng) if _key(cur[g]) != _key(prev[g])]
        hist.append(cur)
        rounds += 1
    return rounds, hist


# ---------------------------------------------------------------- chains
def _chain_levels(kind: str, G: int) -> List[int]:
    if kind == "P":
        return [2 if i % 2 == 0 else 1 for i in range(G)]
    if kind == "K":
        return [3 if i % 2 == 0 else 6 for i in range(G)]
    return [i % 8 for i in range(G)]


def chain(G: int, kind: str) -> Case:
    """See the module docstring.  Nodes h_i = 3i (free 0), a_i = 3i + 1 (edge 1000 to h_i), b_i = 3i + 2 (edge 100);
    every node is a domain of its own at every level but for the pairs / triples of the links."""
    n = 3 * G
    a = lambda i: 3 * i + 1
    rows, cols, ws = [[] for _ in range(n)], [], []
    for i in range(G):
        for v, w in ((3 * i + 1, 1000), (3 * i + 2, 100)):
            rows[3 * i].append((v, w))
            rows[v].append((3 * i, w))
    row_ptr = np.zeros(n + 1, np.int32)
    for v in range(n):
        row_ptr[v + 1] = row_ptr[v] + len(rows[v])
        for u, w in sorted(rows[v]):
            cols.append(u)
            ws.append(w)
    levels = _chain_levels(kind, G)
    n_lv = 8 if kind == "mix" else max(levels) + 1
    parent = [np.arange(n, dtype=np.int64) for _ in range(n_lv)]   # union of the link's nodes per level

    def join(L, x, y):
        p = parent[L]
        rx, ry = p[x], p[y]
        p[p == ry] = rx
    for i in range(1, G):
        link = kind if kind != "mix" else ("P" if i % 2 == 0 else "K")
        join(levels[i] if link == "P" else levels[i - 1], a(i - 1), a(i))
    lv = np.stack([llc.compact(p) for p in parent]).astype(np.int32)
    nd = [int(r.max()) + 1 for r in lv]
    free = np.full(n, 4, np.int32)
    free[0::3] = 0
    topo = synth.Topology(row_ptr, np.asarray(cols, np.int32), np.asarray(ws, np.int32), free, lv[0].copy(),
                          np.full(nd[0], -1, np.int32))
    groups = [Group(gid=1000 + i, roles=[(0, 1, 1, ROLE_EXCLUSIVE)], pair=[[1]], anchors=[(3 * i, 0, 8)],
                    flags=STEP_EXCLUSIVE, level=levels[i]) for i in range(G)]
    return Case(f"chain_{kind}{G}", topo, lv, nd, np.zeros((0, 3), np.int32), _blob(groups), rounds=G,
                tags={"chain", f"chain_{kind}"}, extra=dict(groups=groups, a=[a(i) for i in range(G)],
                                                            b=[a(i) + 1 for i in range(G)]))


def chain_facts(c: Case, replay: bool = True) -> dict:
    """The alternation a, b, a, ..., what removing the chain's term does, and (replay) the replayed round count."""
    G = int(c.blob[2])
    ea, es, ed = expected(c)
    f = dict(alternates=ea.tolist() == [c.extra["a"][i] if i % 2 == 0 else c.extra["b"][i] for i in range(G)],
             all_placed=bool((es == 0).all()), lmask=lmask(c.blob))
    for terms in (("K",), ("P",)):
        f["without_" + "KP"[terms == ("K",)]] = not np.array_equal(expected(c, terms=terms)[0], ea)
    if replay:
        f["rounds"], hist = replay_rounds(c)
        f["replay_final"] = [_key(s) for s in hist[-1]] == [_key(s) for s in states(c)]
        # group i in every round before its own differs from its final placement in the round right before
        f["settles_in_round_i"] = all(_key(hist[i - 1][i]) != _key(hist[-1][i]) for i in range(1, G))
    return f


CHAINS = [(8, "P"), (64, "P"), (8, "K"), (64, "K"), (8, "mix"), (64, "mix")]
REFRESH_CHAIN = (200, "mix")


# ---------------------------------------------------------------- sparse level masks
def _at_levels(case: cg.Case, seed: int, excl_levels, other_levels, n_occ_gids=4) -> Case:
    topo = case.topo
    topo.domain_owner[:] = -1
    lv, nd = llc.partitions47(topo, seed, "random")
    rng = np.random.default_rng(seed + 7)
    groups = [copy.copy(g) for g in case.groups]
    for k, g in enumerate(groups):
        ex = bool(g.flags & STEP_EXCLUSIVE)
        g.level = int(excl_levels[k % len(excl_levels)] if ex else other_levels[k % len(other_levels)])
        if g.fixed_domain >= 0:
            g.fixed_domain = int(rng.integers(0, nd[g.level])) if ex else -1
    gids = sorted({g.gid for g in groups})
    occ = llc.keyed_records(np.random.default_rng(seed + 5), topo.n, gids[:n_occ_gids] + [999], max(1, topo.n // 30),
                            [1, 3, 4, 5, 6, 7])
    return Case(f"{case.name}@{''.join(map(str, excl_levels))}", topo, lv, nd, occ, _blob(groups),
                extra=dict(groups=groups))


SPARSE = [((3, 7), (1, 2, 4, 5, 6)), ((0, 2, 5), (1, 3, 4, 6, 7))]


def sparse_cases() -> List[Case]:
    out = []
    for i, (ex, ot) in enumerate(SPARSE):
        out.append(_at_levels(cg.scarce(400 + i, 517, n_groups=24, exclusive=0.7), 400 + i, ex, ot))
        out.append(_at_levels(cg.scarce(410 + i, 1030, n_groups=20, exclusive=0.6), 410 + i, ex, ot))
    return out


# ---------------------------------------------------------------- level-offset edges
def offsets(n: int = 1024, seed: int = 5) -> Case:
    """Levels 0..7 of partitions47; for L = 0..6 gid 2000 + L claims (L, nd_L - 1) and gid 3000 + L claims
    (L + 1, 0): reported by a one-replica group when L is even, by an idle exclusive group when L is odd.  After them,
    for every claimed domain, a one-replica exclusive group of another gid at another level, anchored on a node of it."""
    topo = synth.make_topology(n, seed=seed, tiers=2, max_free=4)
    topo.domain_owner[:] = -1
    topo.free = np.full(n, 4, np.int32)
    lv, nd = llc.partitions47(topo, seed, "random")
    groups, claims = [], []
    for L in range(7):
        for gid, lvl, d in ((2000 + L, L, nd[L] - 1), (3000 + L, L + 1, 0)):
            groups.append(Group(gid=gid, roles=[(0, 0 if L % 2 else 1, 1, ROLE_EXCLUSIVE)], pair=[[1]], anchors=[],
                                flags=STEP_EXCLUSIVE, fixed_domain=d, level=lvl))
            claims.append((lvl, d))
    rng = np.random.default_rng(seed + 1)
    for k, (lvl, d) in enumerate(claims):
        node = int(rng.choice(np.flatnonzero(lv[lvl] == d)))
        groups.append(Group(gid=4000 + k, roles=[(0, 2, 1, ROLE_EXCLUSIVE)], pair=[[1]], anchors=[(node, 0, 64)],
                            flags=STEP_EXCLUSIVE, level=(lvl + 3) % 8))
    return Case("offsets", topo, lv, nd, np.zeros((0, 3), np.int32), _blob(groups),
                extra=dict(groups=groups, claims=claims))


def offsets_facts(c: Case) -> dict:
    a, s, d = expected(c)
    gr = c.extra["groups"]
    claimed = set()
    for g, grp in enumerate(gr[:14]):
        if d[g] >= 0 or cg.pending(grp) == 0:
            claimed.add((grp.level, grp.fixed_domain))
    boundary = {(L, c.nd[L] - 1) for L in range(7)} | {(L + 1, 0) for L in range(7)}
    readers = {(int(gr[14 + k].level), k) for k in range(14)}
    # every reader's anchor lies in its claimed domain and the claim moves it off that domain's nodes
    moved = []
    no_k = expected(c, terms=("P",))
    off = sum(cg.pending(g) for g in gr[:14])
    for k, (lvl, dm) in enumerate(c.extra["claims"]):
        mine = slice(off + 2 * k, off + 2 * k + 2)
        moved.append(any(c.lv[lvl, x] == dm for x in no_k[0][mine] if x >= 0)
                     and not any(c.lv[lvl, x] == dm for x in a[mine] if x >= 0))
    return dict(claimed_all=claimed == boundary, idle=sum(cg.pending(g) == 0 for g in gr[:14]), moved=moved,
                readers=len(readers), levels=c.lv.shape[0])


# ---------------------------------------------------------------- long pod lists
def pods(n: int = 4096, seed: int = 6) -> Case:
    """Zone level 2 = halves; nodes of zone 0 have free 32, the others 1.  64 hostname-level (level 1) groups of 32
    replicas and 4 of 16 one-replica roles, each fixed to its own node of zone 0, then 4 zone-level groups of 4
    replicas: zone 0 holds 2 112 pods of other gids at level 2."""
    ids = np.arange(n, dtype=np.int64)
    topo = llc.plain_topology(n, ids // 512, free=1, tiers=2)
    zone = (ids >= n // 2).astype(np.int64)
    topo.free[zone == 0] = 32
    lv = np.stack([topo.domain, ids, zone]).astype(np.int32)
    nd = [int(r.max()) + 1 for r in lv]
    rng = np.random.default_rng(seed)
    hosts = rng.choice(n // 2, size=68, replace=False)
    groups = []
    for k in range(64):
        groups.append(Group(gid=5000 + k, roles=[(0, 32, 1, ROLE_EXCLUSIVE)], pair=[[1]], anchors=[],
                            flags=STEP_EXCLUSIVE, fixed_domain=int(hosts[k]), level=1))
    for k in range(4):
        groups.append(Group(gid=5100 + k, roles=[(0, 1, 1, ROLE_EXCLUSIVE)] * 16, pair=np.eye(16, dtype=int).tolist(),
                            anchors=[], flags=STEP_EXCLUSIVE, fixed_domain=int(hosts[64 + k]), level=1))
    for k in range(4):
        groups.append(Group(gid=5200 + k, roles=[(0, 4, 1, ROLE_EXCLUSIVE)], pair=[[1]], anchors=[],
                            flags=STEP_EXCLUSIVE | (STEP_GANG if k % 2 else 0), level=2))
    return Case("pods", topo, lv, nd, np.zeros((0, 3), np.int32), _blob(groups), extra=dict(groups=groups))


def pods_facts(c: Case) -> dict:
    st = states(c)
    on = {}
    for s, L in zip(st, group_levels(c.blob)):
        if s.g.exclusive and s.result()["status"] != 2 and L == 1:
            for m in participating_pods(s):
                on[int(c.lv[2, m])] = on.get(int(c.lv[2, m]), 0) + 1
    a, s, d = result_arrays(st)
    return dict(max_pods=max(on.values()), zone_readers_out=[int(x) for x in d[-4:]],
                without_P=not np.array_equal(expected(c, terms=("K",))[0], a))


# ---------------------------------------------------------------- gids
def gids(n: int = 1024, seed: int = 8) -> Case:
    """partitions47 levels.  Gids 0 (level 3) and 2^31 - 1 (level 5); gid 77 at levels 1 and 6 (the second group
    anchored on the first's node); gids 11 then 12 report domain D of level 6 (fixed) and a later gid-11 group at
    level 6 is fixed to D; records of two gids on one level-2 domain and one level-5 domain block them (-2)."""
    topo = synth.make_topology(n, seed=seed, tiers=2, max_free=4)
    topo.domain_owner[:] = -1
    topo.free = np.full(n, 4, np.int32)
    lv, nd = llc.partitions47(topo, seed, "random")
    rng = np.random.default_rng(seed)
    v = int(rng.integers(0, n))
    D = -1                                                       # set below, away from the first groups' pods
    blk2 = int(lv[2, int(rng.integers(0, n))])
    blk5 = int(lv[5, int(rng.integers(0, n))])
    b2 = np.flatnonzero(lv[2] == blk2)[:1]
    b5 = np.flatnonzero(lv[5] == blk5)[:1]
    occ = np.array([[b2[0], 31, 2], [b2[0], 32, 2], [b5[0], GID_MAX, 5], [b5[0], 0, 5],
                    [int(rng.integers(0, n)), 77, 1]], np.int32)
    one = lambda gid, L, **kw: Group(gid=gid, roles=[(0, 3, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE,
                                     level=L, **kw)
    groups = [one(0, 3), one(GID_MAX, 5), one(77, 1, anchors=[(v, 0, 64)]), one(11, 6, fixed_domain=D),
              one(12, 6, fixed_domain=D), one(77, 6),
              one(11, 6, fixed_domain=D),
              one(0, 7, anchors=[(int(b2[0]), 0, 64)]), one(GID_MAX, 2, anchors=[(int(b5[0]), 0, 64)]),
              Group(gid=GID_MAX, roles=[(0, 2, 1, ROLE_EXCLUSIVE), (1, 2, 1, 0)], pair=[[1, 0], [1, 1]],
                    flags=STEP_EXCLUSIVE | STEP_GANG, level=3)]
    c = Case("gids", topo, lv, nd, occ, _blob(groups[:3]), extra=dict(groups=groups, blocked=(blk2, blk5)))
    a = expected(c)[0]
    p = int(a[6])                                                # the node of the first gid-77 group
    groups[5].anchors = [(p, 0, 64)]                             # the second one wants p's neighbourhood
    used = {int(lv[6, x]) for x in a if x >= 0} | {int(lv[6, v])}
    D = min(set(range(nd[6])) - used - {int(lv[6, b2[0]]), int(lv[6, b5[0]])})
    for g in (3, 4, 6):
        groups[g].fixed_domain = D
    c.blob = _blob(groups)
    c.extra["D"] = D
    return c




def gids_facts(c: Case) -> dict:
    a, s, d = expected(c)
    own = owner(c)
    first = expected(c, reporter="first")
    gr = c.extra["groups"]
    off = [0]
    for g in gr:
        off.append(off[-1] + cg.pending(g))
    seg = lambda g: a[off[g]:off[g + 1]]
    D = c.extra["D"]
    blk2, blk5 = c.extra["blocked"]
    return dict(gid_ends={0, GID_MAX} <= {g.gid for g in gr},
                same_gid_levels=sorted(g.level for g in gr if g.gid == 77),
                shared_gid_matters=not np.array_equal(expected(_regid(c, 2, 78))[0][off[5]:off[6]], seg(5)),
                reporters=[int(d[3]), int(d[4])] == [D, D],
                last_reporter_keeps_out=not any(c.lv[6, x] == D for x in seg(6) if x >= 0),
                first_differs=not np.array_equal(first[0], a),
                blocked=bool((own[2][c.lv[2] == blk2] == lo.BLOCKED).all() and
                             (own[5][c.lv[5] == blk5] == lo.BLOCKED).all()))


def _regid(c: Case, g: int, gid: int) -> Case:
    gb = np.array(c.blob, np.int32, copy=True)
    gb[8 + 12 * g] = gid
    return Case(c.name, c.topo, c.lv, c.nd, c.occ, gb, extra=c.extra)


# ---------------------------------------------------------------- <true> against <false>
def level0_pairs() -> List[tuple]:
    """(unmoved case, moved case): commit_gen batches with records-free partitions47 levels; the moved batch's
    non-exclusive groups sit at levels 1 + g % 7 with their fixed domains dropped (kept when they are -1)."""
    out = []
    for i, base in enumerate([cg.chain(16, 16, 2), cg.gang_frees(), cg.domain_move(0), cg.table_reads(0),
                              cg.domains(0), cg.domains(1), cg.scarce(0, 40), cg.scarce(3, 40),
                              cg.scarce(21, 31, n_groups=16), cg.scarce(23, 4097, n_groups=16)]):
        if not any(not g.flags & STEP_EXCLUSIVE for g in base.groups):
            continue
        topo = base.topo
        lv, nd = llc.partitions47(topo, 500 + i, "random")
        occ = np.zeros((0, 3), np.int32)
        g0 = [copy.copy(g) for g in base.groups]
        for g in g0:
            g.level = 0
        moved = [copy.copy(g) for g in g0]
        for k, g in enumerate(moved):
            if not g.flags & STEP_EXCLUSIVE:
                g.level = 1 + k % 7
                g.fixed_domain = -1 if g.fixed_domain >= nd[g.level] else g.fixed_domain
        out.append((Case(base.name, topo, lv, nd, occ, _blob(g0), rounds=base.rounds, extra=dict(groups=g0)),
                    Case(base.name + "@moved", topo, lv, nd, occ, _blob(moved), rounds=base.rounds,
                         extra=dict(groups=moved))))
    return out


# ---------------------------------------------------------------- the whole seed set
def cases() -> List[Case]:
    return ([chain(G, k) for G, k in CHAINS] + sparse_cases() + [offsets(), pods(), gids()])


BULLETS = ("chain_P", "chain_K", "chain_mix", "lmask_ff", "sparse_37", "sparse_025", "offsets", "idle_offsets",
           "long_pod_list", "gid_ends", "shared_gid_levels", "two_reporters", "blocked_records", "gang_vanishes_lv",
           "claim_moves_lv", "n_ge_1000")


def coverage(cs: List[Case], snap: Dict[str, list], comm: Dict[str, list]) -> Dict[str, bool]:
    """Which bullets the cases reach.  snap[name] / comm[name]: per group (assign, status, domain) of round 1 (every
    group against the snapshot) and of the committed oracle."""
    c = dict.fromkeys(BULLETS, False)
    for case in cs:
        for t in case.tags & set(BULLETS):
            c[t] = True
        m = lmask(case.blob)
        c["lmask_ff"] |= m == 0xFF
        c["sparse_37"] |= m == (1 << 3 | 1 << 7)
        c["sparse_025"] |= m == (1 << 0 | 1 << 2 | 1 << 5)
        c["offsets"] |= case.name == "offsets"
        c["idle_offsets"] |= case.name == "offsets" and any(cg.pending(g) == 0 for g in case.extra["groups"])
        c["long_pod_list"] |= case.name == "pods"
        c["n_ge_1000"] |= case.topo.n >= 1000
        gr = case.extra["groups"]
        c["gid_ends"] |= {0, GID_MAX} <= {g.gid for g in gr}
        lv_of = {}
        for g in gr:
            if g.flags & STEP_EXCLUSIVE:
                lv_of.setdefault(g.gid, set()).add(g.level)
        c["shared_gid_levels"] |= any(len(x) >= 2 for x in lv_of.values())
        c["blocked_records"] |= bool((owner(case) == lo.BLOCKED).any())
        if case.name not in comm:
            continue
        rep = {}
        for g, (grp, (sa, ss, sd), (ca, cs_, cd)) in enumerate(zip(gr, snap[case.name], comm[case.name])):
            if grp.level >= 1 and cg.pending(grp) > 0:
                c["gang_vanishes_lv"] |= bool(grp.flags & STEP_GANG) and ss == 0 and cs_ == 2
                c["claim_moves_lv"] |= any(x >= 0 and y >= 0 and x != y for x, y in zip(sa, ca))
            if grp.flags & STEP_EXCLUSIVE and cd >= 0 and cs_ != 2:
                rep.setdefault((grp.level, cd), set()).add(grp.gid)
        c["two_reporters"] |= any(len(x) >= 2 for x in rep.values())
    return c
