"""Seeded generator of committed batches (rbgtopo_place_groups_committed, DESIGN.md §3.8; test infrastructure).

tests/groups_gen.py reaches the limits of the GROUPS ABI; this file adds what only a committed batch has — the rounds
of k_plan_group_commit and the claim lists they read:
  * full chains: G identical one-replica groups on nodes of capacity 1, every group's node depends on the one before,
    so the call takes exactly G rounds (G = 64, and a chain with no idle group, on the host's `rounds >= n_groups`
    bound);
  * claims that move or vanish: under scarce capacity a gang group placed in round 1 fails once the earlier claims
    appear and frees nodes later groups read as full; a non-gang group moves between rounds;
  * domain claims: several exclusive groups of one gid report the same fixed domain, two gids report one domain and
    only the last reporter keeps a later group of the first gid out (`two_reporters`), reported
    domains that change between rounds (one seen by a later group only through the domain), idle exclusive groups with a fixed domain (claims before round 0), opted-out
    roles inside exclusive groups;
  * long claim lists: a hub of free = 32 767 that hundreds of groups' replicas land on, the claims summing exactly to
    its capacity, demand-0 replicas that still link a claim;
  * claims read through the table of patched nodes: groups anchored next to the claimed nodes (which sit deep in the
    background order), multi-wave and 16-role groups;
  * N in {1, 31, 130, 4097}.
`coverage()` reports which of these a set of cases reached, from the blobs and the oracle's results (the chains'
exact round counts are asserted by the GPU tests).  Every group passes
groups_gen.exact_ok."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional

import numpy as np

import groups_gen as gg
import levels_oracle as lo
from rbg_b200 import synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, STEP_GANG, Group, GroupsBuilder

HUB_FREE = 32767


@dataclass
class Case:
    name: str
    topo: synth.Topology
    groups: List[Group]
    blob: np.ndarray
    rounds: Optional[int] = None          # the exact number of rounds, where the construction fixes it
    tags: set = field(default_factory=set)


def build(groups: List[Group]) -> np.ndarray:
    gb = GroupsBuilder()
    for g in groups:
        gb.add(g)
    return gb.build()


def _fit(grp: Group, row_w: int) -> Group:
    """Lower the heaviest pair weight until the group is under the exactness bound."""
    while not gg.exact_ok(grp, row_w):
        p = np.asarray(grp.pair)
        p[np.unravel_index(int(np.argmax(p)), p.shape)] -= 1
        grp.pair = p.tolist()
    return grp


def _case(name, topo, groups, rounds=None, tags=()):
    row_w = gg.wsum_max(topo)
    groups = [_fit(g, row_w) for g in groups]
    return Case(name, topo, groups, build(groups), rounds, set(tags))


def pending(g: Group) -> int:
    return sum(r[1] for r in g.roles)


def chain(n_groups: int, n_nodes: int, seed: int = 0, idle_every: int = 0) -> Case:
    """n_groups one-replica demand-1 groups on nodes of capacity 1 (n_nodes >= n_groups): round r settles group r - 1,
    so the call takes exactly n_groups rounds.  idle_every > 0 puts an idle group after every idle_every-th one."""
    assert n_nodes >= n_groups
    topo = synth.make_topology(n_nodes, seed=seed, tiers=2, max_free=1)
    topo.free = np.ones(n_nodes, dtype=np.int32)
    groups = []
    for i in range(n_groups):
        groups.append(Group(gid=500 + i, roles=[(0, 1, 1, ROLE_EXCLUSIVE)], pair=[[1]], anchors=[], flags=0))
        if idle_every and i % idle_every == idle_every - 1:
            groups.append(Group(gid=900 + i, roles=[(0, 0, 1, ROLE_EXCLUSIVE)], pair=[[1]], anchors=[], flags=0))
    tags = {"chain"} | ({"chain_64"} if n_groups >= 64 else set()) | \
        ({"chain_n0_eq_ng"} if not idle_every else {"chain_idle"})
    return _case(f"chain{n_groups}/{n_nodes}", topo, groups, rounds=n_groups, tags=tags)


def scarce(seed: int, n_nodes: int, n_groups: int = 24, exclusive: float = 0.3) -> Case:
    """Many small groups, gang and not, under scarce capacity: claims move and vanish between rounds."""
    rng = np.random.default_rng(seed)
    topo = synth.make_topology(n_nodes, seed=seed + 3, tiers=2, owned_frac=0.2 if n_nodes >= 16 else 0.0, max_free=2)
    topo.free = np.where(rng.random(n_nodes) < 0.5, 0, topo.free).astype(np.int32)
    if n_nodes == 1 or not topo.free.any():
        topo.free[0] = 2
    n_dom = len(topo.domain_owner)
    groups = []
    for g in range(n_groups):
        q = int(rng.integers(1, 4))
        lv = np.sort(rng.integers(0, 2, size=q))
        roles = [(int(lv[i]), int(rng.integers(0, 4)), int(rng.choice([0, 1, 1, 2])),
                  ROLE_EXCLUSIVE if rng.random() < 0.8 else 0) for i in range(q)]
        pair = rng.integers(0, 3, size=(q, q))
        np.fill_diagonal(pair, 1)
        excl = rng.random() < exclusive
        gid = 300 + (int(rng.integers(0, g)) if g and rng.random() < 0.2 else g)
        fixed = int(rng.integers(0, n_dom)) if excl and rng.random() < 0.2 else -1
        anchors = [(int(rng.integers(0, n_nodes)), int(rng.integers(0, q)), 1) for _ in range(int(rng.integers(0, 3)))]
        groups.append(Group(gid=gid, roles=roles, pair=pair.tolist(), anchors=anchors,
                            flags=(STEP_EXCLUSIVE if excl else 0) | (STEP_GANG if rng.random() < 0.5 else 0),
                            fixed_domain=fixed))
    return _case(f"scarce{seed}/{n_nodes}", topo, groups)


def gang_frees() -> Case:
    """Two nodes of capacity 1.  Group 0 takes the best node; the gang group 1 takes both in round 1 and fails in
    round 2, which frees the second node group 2 read as full: only the old-node term of k_commit_diff re-runs it."""
    topo = synth.make_topology(2, seed=1, tiers=1, max_free=1)
    topo.free = np.ones(2, dtype=np.int32)
    one = dict(pair=[[1]], anchors=[])
    groups = [Group(gid=1, roles=[(0, 1, 1, 0)], flags=0, **one),
              Group(gid=2, roles=[(0, 2, 1, 0)], flags=STEP_GANG, **one),
              Group(gid=3, roles=[(0, 1, 1, 0)], flags=0, **one)]
    return _case("gang_frees", topo, groups, rounds=3)


def domains(seed: int, n_nodes: int = 96) -> Case:
    """Exclusive groups racing for few domains: idle groups with a fixed domain (claims before round 0), several groups
    of one gid reporting the same fixed domain, shared gids, opted-out roles, scarce capacity so that reported domains
    change between rounds."""
    rng = np.random.default_rng(seed)
    topo = synth.make_topology(n_nodes, seed=seed + 5, tiers=2, max_free=2)
    topo.domain_owner[:] = -1
    topo.free = np.where(rng.random(n_nodes) < 0.4, 0, topo.free).astype(np.int32)
    n_dom = len(topo.domain_owner)
    d_shared = int(rng.integers(0, n_dom))
    groups = []
    for i in range(2):                                          # idle, exclusive, fixed domain
        groups.append(Group(gid=700 + i, roles=[(0, 0, 1, ROLE_EXCLUSIVE)], pair=[[1]], anchors=[],
                            flags=STEP_EXCLUSIVE, fixed_domain=int(rng.integers(0, n_dom))))
    for g in range(18):
        q = int(rng.integers(1, 4))
        lv = np.sort(rng.integers(0, 2, size=q))
        roles = [(int(lv[i]), int(rng.integers(1, 4)), int(rng.choice([1, 1, 2])),
                  ROLE_EXCLUSIVE if (i > 0 or q == 1) and rng.random() < 0.8 else 0) for i in range(q)]
        pair = rng.integers(0, 3, size=(q, q))
        np.fill_diagonal(pair, 1)
        if g % 6 == 0:                                          # three reporters of one gid and one fixed domain
            groups.append(Group(gid=777, roles=roles, pair=pair.tolist(), anchors=[], flags=STEP_EXCLUSIVE,
                                fixed_domain=d_shared))
            continue
        gid = 710 + (int(rng.integers(0, 4)) if rng.random() < 0.3 else g)
        groups.append(Group(gid=gid, roles=roles, pair=pair.tolist(), anchors=[],
                            flags=STEP_EXCLUSIVE | (STEP_GANG if rng.random() < 0.3 else 0),
                            fixed_domain=int(rng.integers(0, n_dom)) if rng.random() < 0.15 else -1))
    return _case(f"domains{seed}/{n_nodes}", topo, groups)


def hub(seed: int = 0, n_nodes: int = 256) -> Case:
    """Node 0 has free = 32 767, every other node 0: 341 groups of 32 demand-3 replicas and one of 31 demand-1 replicas
    fill it exactly, groups of demand-0 replicas in between still link claims; the groups after the fill point find
    it full (one more replica does not fit)."""
    topo = synth.make_topology(n_nodes, seed=seed, tiers=2, max_free=1)
    topo.free = np.zeros(n_nodes, dtype=np.int32)
    topo.free[0] = HUB_FREE
    groups = []
    for i in range(341):
        groups.append(Group(gid=1000 + i, roles=[(0, 32, 3, 0)], pair=[[1]], anchors=[], flags=0))
        if i % 60 == 30:
            groups.append(Group(gid=5000 + i, roles=[(0, 32, 0, 0)], pair=[[1]], anchors=[], flags=0))
    assert 341 * 32 * 3 + 31 == HUB_FREE
    groups.append(Group(gid=2000, roles=[(0, 31, 1, 0)], pair=[[1]], anchors=[], flags=0))
    groups.append(Group(gid=2001, roles=[(0, 1, 1, 0)], pair=[[1]], anchors=[], flags=0))
    groups.append(Group(gid=2002, roles=[(0, 2, 1, 0)], pair=[[1]], anchors=[], flags=STEP_GANG))
    groups.append(Group(gid=2003, roles=[(0, 3, 0, 0)], pair=[[1]], anchors=[], flags=0))
    return _case(f"hub/{n_nodes}", topo, groups)


def table_reads(seed: int = 0, n_nodes: int = 512) -> Case:
    """Claims read through the table of patched nodes: node a is full and anchors every group; its NVLink peers have
    capacity 1 and sit deep in the background order (every other node has capacity 4), so only a group's table shows
    them.  One-replica groups chain through the peers; two-level groups place their second wave next to the first;
    a 16-role group (groups_gen) reads its whole neighbourhood through the table."""
    rng = np.random.default_rng(seed)
    topo = synth.make_topology(n_nodes, seed=seed + 9, tiers=2, max_free=4)
    a = int(rng.integers(0, n_nodes // 8)) * 8
    peers = topo.col_idx[topo.row_ptr[a]:topo.row_ptr[a + 1]]
    peers = peers[topo.edge_w[topo.row_ptr[a]:topo.row_ptr[a + 1]] == 1000]
    free = np.full(n_nodes, 4, dtype=np.int32)
    free[peers] = 1
    free[a] = 0
    topo.free = free
    groups = []
    for i in range(len(peers) + 2):
        groups.append(Group(gid=600 + i, roles=[(0, 1, 1, 0)], pair=[[1]], anchors=[(a, 0, 64)], flags=0))
    for i in range(6):                                          # two waves: the second is anchored on the first
        groups.append(Group(gid=650 + i, roles=[(0, 1, 1, 0), (1, 2, 1, 0)], pair=[[1, 0], [8, 1]],
                            anchors=[(a, 0, 16)], flags=STEP_GANG if i % 2 else 0))
    wide = gg._wide(rng, 5)
    groups.append(Group(gid=680, roles=wide, pair=gg._pair(rng, len(wide), False), anchors=[(a, 0, 4)], flags=0))
    return _case(f"table/{n_nodes}", topo, groups)


def domain_move(seed: int = 0, n_nodes: int = 512) -> Case:
    """A reported domain that changes between rounds, seen by a later exclusive group only through the domain.
    W (plain) and X (exclusive) are anchored on the full node a and want p, the one peer of a's NVLink domain D with
    room for demand 2; W takes it, so X moves in round 2 to a neighbour q of a outside D.  Y (exclusive, demand 1) is
    anchored on b, whose only usable neighbour is m in D: it read D through m in round 2, while X's claim was there.
    p and q sit deep in the background order and outside Y's table, so only X's changed domain re-runs Y (3 rounds)."""
    topo = synth.make_topology(n_nodes, seed=seed + 13, tiers=2, max_free=4)
    topo.domain_owner[:] = -1
    rp, col, dom = topo.row_ptr, topo.col_idx, topo.domain
    nb = lambda v: set(int(x) for x in col[rp[v]:rp[v + 1]])
    for a in range(0, n_nodes, 8):
        peers = [v for v in nb(a) if dom[v] == dom[a]]
        cross_a = {v for v in nb(a) if dom[v] != dom[a]}
        for m in peers:
            for b in sorted(v for v in nb(m) if dom[v] != dom[a] and v not in cross_a):
                others = [v for v in peers if v != m and v not in nb(b)]
                if others and not (nb(b) & cross_a) and a not in nb(b):
                    p = others[0]
                    free = np.full(n_nodes, 4, dtype=np.int32)
                    free[dom == dom[a]] = 1
                    free[a] = 0
                    free[p] = 2
                    free[list(cross_a)] = 2
                    free[dom == dom[b]] = 0
                    free[[v for v in nb(b) if v != m]] = 0
                    topo.free = free
                    groups = [Group(gid=1, roles=[(0, 1, 2, 0)], pair=[[1]], anchors=[(a, 0, 700)], flags=0),
                              Group(gid=2, roles=[(0, 1, 2, ROLE_EXCLUSIVE)], pair=[[1]], anchors=[(a, 0, 700)],
                                    flags=STEP_EXCLUSIVE),
                              Group(gid=3, roles=[(0, 1, 1, ROLE_EXCLUSIVE)], pair=[[1]], anchors=[(b, 0, 700)],
                                    flags=STEP_EXCLUSIVE)]
                    assert all(gg.exact_ok(g, gg.wsum_max(topo)) for g in groups)
                    return _case(f"domain_move/{n_nodes}", topo, groups, rounds=3)
    raise AssertionError("no such nodes")


def two_reporters(seed: int = 0, n_nodes: int = 64) -> Case:
    """Two gids report one domain D: gid 11, then gid 12 with fixed_domain = D.  D holds the head of the background
    order, which a later gid-11 group wants: only the last reporter's gid (12) keeps it out."""
    from topo_gen import base_ref, key_node, order_ref
    topo = synth.make_topology(n_nodes, seed=seed + 17, tiers=2, max_free=4)
    topo.domain_owner[:] = -1
    topo.free = np.full(n_nodes, 4, dtype=np.int32)
    d = int(topo.domain[key_node(order_ref(base_ref(topo)))[0]])
    one = dict(roles=[(0, 1, 1, ROLE_EXCLUSIVE)], pair=[[1]], anchors=[], flags=STEP_EXCLUSIVE)
    groups = [Group(gid=11, fixed_domain=d, **one), Group(gid=12, fixed_domain=d, **one), Group(gid=11, **one)]
    return _case(f"two_reporters/{n_nodes}", topo, groups)


def extremes(seed: int) -> List[Case]:
    return [scarce(seed + i, n, n_groups=16 if n > 1 else 6) for i, n in enumerate((1, 31, 130, 4097))]


def occupancy(case: Case, seed: int, n_levels: int = 7):
    """Records at every level for a case: partitions from levels_oracle.random_levels (nested and crossing), records
    of the batch's own gids (shared) and of one gid outside it.  Returns (level_domain [L+1][n], occ, owner0)."""
    rng = np.random.default_rng(seed)
    lv = lo.random_levels(rng, case.topo.n, case.topo.domain, n_levels,
                          [True, False, True, False, True, False, True][:n_levels])
    gids = sorted({g.gid for g in case.groups})
    occ = lo.random_occ(rng, case.topo.n, n_levels, gids[:4] + [99999], max(1, case.topo.n // 6))
    return lv, occ, lo.derive_level_owner(lv, occ)[0]


def occupancy_cases():
    """Exclusive batches with records at 3 and 7 levels above level 0, nested and crossing partitions."""
    out = []
    for i, case in enumerate([domains(40), domains(41, 130), scarce(42, 33, exclusive=0.7), scarce(43, 130, exclusive=0.7)]):
        lv, occ, owner0 = occupancy(case, 50 + i, n_levels=7 if i % 2 else 3)
        out.append((case, lv, occ, owner0))
    # two gids reporting one domain, with records on nested levels outside that domain: the domain stays usable by
    # its reporters' gids, so only the last reporter keeps the later gid-11 group out
    case = two_reporters(1)
    rng = np.random.default_rng(54)
    lv = lo.random_levels(rng, case.topo.n, case.topo.domain, 2, [True, True])
    d = case.groups[0].fixed_domain
    occ = lo.random_occ(rng, case.topo.n, 2, [11, 12, 99], 12)
    occ = occ[case.topo.domain[occ[:, 0]] != d]
    out.append((case, lv, occ, lo.derive_level_owner(lv, occ)[0]))
    return out


def known_occupancy():
    """The 4-node known answer of DESIGN.md §3.9: level-0 domains [0, 0, 1, 1], level 1 [1, 0, 0, 1], one record
    (node 2, gid 9, level 1) — owner_0 = [-1, 9, 9, 9].  Two exclusive one-replica groups of gid 7 on nodes of capacity
    1: the first takes node 0 and reports domain 0; node 1 stays blocked for the second."""
    row_ptr = np.array([0, 1, 3, 5, 6], dtype=np.int32)
    col = np.array([1, 0, 2, 1, 3, 2], dtype=np.int32)
    w = np.array([1000, 1000, 100, 100, 10, 10], dtype=np.int32)
    topo = synth.Topology(row_ptr, col, w, np.ones(4, dtype=np.int32), np.array([0, 0, 1, 1], dtype=np.int32),
                          np.full(2, -1, dtype=np.int32))
    lv = np.array([[0, 0, 1, 1], [1, 0, 0, 1]], dtype=np.int32)
    occ = np.array([[2, 9, 1]], dtype=np.int32)
    groups = [Group(gid=7, roles=[(0, 1, 1, ROLE_EXCLUSIVE)], pair=[[1]], anchors=[], flags=STEP_EXCLUSIVE)
              for _ in range(2)]
    return topo, lv, occ, groups, build(groups)


def cases(seed_base: int = 0) -> List[Case]:
    """The seed set of the GPU tests."""
    out = [chain(64, 96, seed_base), chain(40, 64, seed_base + 1, idle_every=5), chain(16, 16, seed_base + 2),
           gang_frees(), domain_move(seed_base), two_reporters(seed_base), hub(seed_base), table_reads(seed_base)]
    out += [domains(seed_base + s) for s in range(4)]
    out += [scarce(seed_base + s, 40) for s in range(6)]
    out += extremes(seed_base + 20)
    return out


BULLETS = ("chain_64", "chain_n0_eq_ng", "chain_idle", "gang_vanishes", "claim_moves", "old_node", "shared_reporters",
           "last_reporter_wins", "domain_moves", "idle_fixed", "opt_out", "hub_long_list", "hub_exact_full",
           "demand0_claim", "table_reads", "multi_wave", "wide_16", "n_1", "n_31", "n_130", "n_4097")


def placements(s):
    """(role index, node, demand) of every pending replica of a group's oracle state, in GROUPS-blob order."""
    nodes = s.result()["nodes"]
    return [(ri, nodes[f"{s.g.name}-{s.g.roles[ri].name}-{s.first[ri] + c}"], s.g.roles[ri].demand)
            for ri in s.order for c in range(s.pending[ri])]


def coverage(cs: List[Case], results: Dict[str, tuple]) -> Dict[str, bool]:
    """Which bullets the cases reach.  results[name] = (committed states, snapshot states) of the oracle.  Outside the
    chains (whose round counts the GPU tests assert) every bullet is read off the blob or the oracle's results.  A
    group's snapshot result is its round-1 result (in a batch without idle exclusive groups): where its committed
    result differs, claims moved or vanished under it."""
    from topo_gen import base_ref, order_ref, pos_ref
    c = dict.fromkeys(BULLETS, False)
    for case in cs:
        for t in case.tags & set(BULLETS):
            c[t] = True
        n = case.topo.n
        c["n_1"] |= n == 1
        c["n_31"] |= n == 31
        c["n_130"] |= n == 130
        c["n_4097"] |= n == 4097
        for g in case.groups:
            if g.flags & STEP_EXCLUSIVE:
                c["opt_out"] |= any(r[1] > 0 and not r[3] & ROLE_EXCLUSIVE for r in g.roles)
                c["idle_fixed"] |= pending(g) == 0 and g.fixed_domain >= 0
        if case.name not in results:
            continue
        comm, snap = results[case.name]
        pos = pos_ref(order_ref(base_ref(case.topo)))
        rp, col = case.topo.row_ptr, case.topo.col_idx
        pc = [placements(s) for s in comm]
        ps = [placements(t) for t in snap]
        used = np.zeros(n, dtype=np.int64)
        on = np.zeros(n, dtype=np.int64)
        for pl in pc:
            for _, x, dem in pl:
                if x >= 0:
                    used[x] += dem
                    on[x] += 1
        reporters = {}                                          # domain -> gids of its reporters, in group order
        for h, (g, s, t) in enumerate(zip(case.groups, comm, snap)):
            rc, rt = s.result(), t.result()
            ch, sh = {x for _, x, _ in pc[h] if x >= 0}, {x for _, x, _ in ps[h] if x >= 0}
            earlier_c = set().union(*[{x for _, x, _ in pc[k] if x >= 0} for k in range(h)])
            earlier_s = set().union(*[{x for _, x, _ in ps[k] if x >= 0} for k in range(h)])
            c["gang_vanishes"] |= bool(g.flags & STEP_GANG) and rt["status"] == 0 and rc["status"] == 2 and pending(g) > 0
            c["claim_moves"] |= not g.flags & STEP_GANG and any(
                x >= 0 and y >= 0 and x != y for (_, x, _), (_, y, _) in zip(pc[h], ps[h]))
            # a node an earlier group held in round 1 but not in the end, which this group then uses
            c["old_node"] |= bool(ch & (earlier_s - earlier_c))
            # an earlier group's claim moved this group off a node it read only through its table: a neighbour of
            # its scheduled pods outside the background order's first warp-load
            table = set(int(v) for a in g.anchors for v in list(col[rp[a[0]]:rp[a[0] + 1]]) + [a[0]])
            c["table_reads"] |= any(x in table and pos[x] >= 32 and x not in ch for x in sh & earlier_c)
            c["multi_wave"] |= len(gg.waves_of(g.roles)) >= 2 and len(ch - sh) > 0
            c["wide_16"] |= len(g.roles) == 16 and len(ch) > 0
            c["demand0_claim"] |= any(dem == 0 and x >= 0 and used[x] == case.topo.free[x] > 0 for _, x, dem in pc[h])
            if g.flags & STEP_EXCLUSIVE:
                if rc["domain"] >= 0 and rc["status"] != 2:
                    c["domain_moves"] |= rt["domain"] >= 0 and rt["domain"] != rc["domain"] and pending(g) > 0
                # a domain whose last reporter is another gid than an earlier reporter of this group's gid, which this
                # group took in round 1 and gave up
                gids = reporters.get(rt["domain"], [])
                c["last_reporter_wins"] |= g.gid in gids[:-1] and gids[-1] != g.gid and rc["domain"] != rt["domain"]
                if rc["domain"] >= 0 and rc["status"] != 2:
                    reporters.setdefault(rc["domain"], []).append(g.gid)
        c["shared_reporters"] |= any(len(v) >= 2 for v in reporters.values())
        full = (used == case.topo.free) & (case.topo.free >= HUB_FREE)
        c["hub_long_list"] |= bool((on >= 256).any())
        c["hub_exact_full"] |= bool(full.any()) and any(
            x < 0 and dem > 0 for pl in pc for _, x, dem in pl)
    return c
