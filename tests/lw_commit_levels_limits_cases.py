"""Committed leader-worker batches at exclusive levels at their limits (DESIGN.md §3.16; test infrastructure), for the
claim lists LwLists::build relinks every round, commit_owner<true> inside mixed emit blocks, and the ranked replay of
k_alternates_commit_coloc_lv.

Every builder returns a Case (snapshot, GROUPS blob groups, (S, C) table, level partitions, records and, where the
construction pins it, the round count) and a *_facts function gives the facts its precondition needs;
tests/test_oracle_lw_committed_levels_limits.py asserts them on the oracle alone and
tests/test_gpu_lw_committed_levels_limits.py places the cases on the device.

replay         §3.13 / §3.16's host loop on the oracle: round 1 runs every group against no claims; a round runs the
               groups >= lo against the claims the previous round left ((node, demand), the reported (level, domain,
               gid) and the nodes of placed participating pods); the next round starts at cmin + 1, cmin = the lowest
               group whose claims changed.  Per round it reports the (L, d) pod lists and domain lists the device holds.
churn_*        a list present in round r and gone (or shorter) in round r + 1, and a later group that reads its domain.
final_lists    claims only the final lists carry: ranking with the last round's lists gives other alternates.
chain          G groups of two-pod replicas, each a claim away from the next: exactly G rounds, through 'P', 'K' or
               both at all eight levels ('mix').
levels         all eight levels (lmask 0xFF) with co-location 7 / exclusive 3 and the reverse, and the sparse masks.
offsets        for every adjacent level pair, domain nd_L - 1 of L and domain 0 of L + 1, claimed by reporters, by pods
               or by idle fixed groups, each read by a later group anchored inside it.
long_*         2 048 hostname-keyed pods in one zone (nesting and non-nesting zones) read by zone-keyed groups.
opted_out, gang_mid_chain, gids, emit_blocks, ragged_*, scale cases: see their builders."""
from __future__ import annotations

import dataclasses
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

import numpy as np

import levels_limits_cases as llc
import levels_oracle as lo
import lw_commit_gen as lg
import lw_commit_levels_gen as lvg
import lw_committed_oracle as lco
import lw_oracle as lw
from lw_committed_levels_oracle import FREE, group_claims, place_group, run_lw_committed_levels_ranked
from rbg_b200 import synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, STEP_GANG, Group

GID_MAX = (1 << 31) - 1


@dataclass
class Case(lvg.LvFleet):
    name: str = ""
    rounds: Optional[int] = None
    tags: set = field(default_factory=set)
    extra: dict = field(default_factory=dict)

    def owner(self) -> np.ndarray:
        return lo.derive_level_owner_fast(self.lv, self.occ) if self.topo.n > 50_000 else super().owner()

    def expected_ranked(self, n_alt: int, claims=None):
        return run_lw_committed_levels_ranked(self.topo, self.blob(), self.role_pods(), n_alt, self.lv, self.owner(),
                                              self.nd, claims=claims)

    def replace(self, **kw) -> "Case":
        return dataclasses.replace(self, **kw)


def lmask(groups) -> int:
    return sum({1 << g.level for g in groups if g.flags & STEP_EXCLUSIVE})


def pod_offsets(c: Case) -> List[int]:
    """First pod of every group, and the total."""
    out = [0]
    for g, rp in zip(c.groups, c.rp):
        out.append(out[-1] + sum(r[1] * s for r, (s, _) in zip(g.roles, rp)))
    return out


# ---------------------------------------------------------------- the round replay
@dataclass
class Round:
    lo: int
    assign: np.ndarray
    status: np.ndarray
    domain: np.ndarray
    claims: list                 # per group (cap, reported domain, participating pods) after the round
    pod_lists: Dict[tuple, int]  # (L, d) -> entries of the pod lists the round read
    dom_lists: Dict[tuple, int]  # (L, d) -> entries of the domain lists the round read


NONE = ({}, -1, [])


def _fresh(c: Case):
    gb, rp = c.blob(), c.role_pods()
    spans, r0 = [], 0
    for X in lco.groups_of(gb, rp):
        spans.append((r0, X.q, X.pod0))
        r0 += X.q
    gbi, rpi = np.asarray(gb, np.int64), np.asarray(rp, np.int64).reshape(-1, 2)
    return lambda g: lw.LwGroup(gbi, g, rpi[spans[g][0]:spans[g][0] + spans[g][1]], spans[g][2])


def lists_of(c: Case, claims) -> tuple:
    """The (L, d) pod lists and domain lists LwLists::build links from `claims`."""
    m = lmask(c.groups)
    pl, dl = {}, {}
    for g, (cap, rep, pods) in enumerate(claims):
        lh = c.groups[g].level
        if rep >= 0:
            dl[(lh, rep)] = dl.get((lh, rep), 0) + 1
        for node in pods:
            for L in range(8):
                if m >> L & 1 and L != lh:
                    k = (L, int(c.lv[L][node]))
                    pl[k] = pl.get(k, 0) + 1
    return pl, dl


def claims_view(c: Case, claims, upto: Optional[int] = None):
    """(claimed, last, pods) the groups before `upto` leave in `claims` (last reporter of a domain wins)."""
    claimed, pods = {}, []
    last = [np.full(int(k), FREE, np.int32) for k in c.nd]
    for h, (cap, rep, mine) in enumerate(claims[:upto]):
        for node, amt in cap.items():
            claimed[node] = claimed.get(node, 0) + amt
        L = c.groups[h].level
        if rep >= 0:
            last[L][rep] = c.groups[h].gid
        pods += [(c.groups[h].gid, L, m) for m in mine]
    return claimed, last, pods


def rerun(c: Case, g: int, claims, fresh=None, own=None):
    """Group g placed against `claims` of the groups before it: (its pods, status, domain)."""
    fresh = fresh or _fresh(c)
    own = c.owner() if own is None else own
    X = fresh(g)
    assign = np.full(pod_offsets(c)[-1], -1, np.int32)
    claimed, last, pods = claims_view(c, claims, g)
    other = lo.unused_gid({x.gid for x in c.groups})
    s, d = place_group(c.topo, np.asarray(c.lv), own, c.nd, X, c.groups[g].level, claimed, last, pods, other, assign)
    return assign[X.pod0:X.pod0 + X.n_pods].copy(), int(s), int(d)


def replay(c: Case) -> List[Round]:
    """The rounds of the call (module docstring); the last round's results are the call's."""
    fresh = _fresh(c)
    own = c.owner()
    dom = np.asarray(c.lv)
    ng = len(c.groups)
    other = lo.unused_gid({x.gid for x in c.groups})
    claims = [NONE] * ng
    assign = np.full(pod_offsets(c)[-1], -1, np.int32)
    status = np.full(ng, -9, np.int32)
    domain = np.full(ng, -9, np.int32)
    out, lo_g = [], 0
    while True:
        pl, dl = lists_of(c, claims)
        claimed, last, pods = {}, [np.full(int(k), FREE, np.int32) for k in c.nd], []
        Xs = {}
        for g in range(ng):
            L = c.groups[g].level
            if g >= lo_g:
                X = Xs[g] = fresh(g)
                assign[X.pod0:X.pod0 + X.n_pods] = -1
                status[g], domain[g] = place_group(c.topo, dom, own, c.nd, X, L, claimed, last, pods, other, assign)
            cap, rep, mine = claims[g]           # what the round reads: the previous round's claims
            for node, amt in cap.items():
                claimed[node] = claimed.get(node, 0) + amt
            if rep >= 0:
                last[L][rep] = c.groups[g].gid
            pods += [(c.groups[g].gid, L, m) for m in mine]
        cmin = None
        new = list(claims)
        for g in range(lo_g, ng):
            cap, rep, mine = group_claims(Xs[g], assign, status[g], domain[g])
            new[g] = (cap, rep, sorted(mine))
            if cmin is None and (new[g][0] != claims[g][0] or new[g][1:] != (claims[g][1], sorted(claims[g][2]))):
                cmin = g
        claims = new
        out.append(Round(lo_g, assign.copy(), status.copy(), domain.copy(), list(claims), pl, dl))
        if cmin is None or cmin + 1 >= ng:
            return out
        lo_g = cmin + 1


def key(r: Round) -> tuple:
    return r.assign.tolist(), r.status.tolist(), r.domain.tolist()


# ---------------------------------------------------------------- hand-built graphs
def graph(n: int, edges, free, lv, nd=None) -> tuple:
    """(topology, lv, nd): the given weighted edges, free per node, partitions (row 0 = the snapshot's domain)."""
    rows = [[] for _ in range(n)]
    for u, v, w in edges:
        rows[u].append((v, w))
        rows[v].append((u, w))
    row_ptr = np.zeros(n + 1, np.int32)
    cols, ws = [], []
    for v in range(n):
        row_ptr[v + 1] = row_ptr[v] + len(rows[v])
        for u, w in sorted(rows[v]):
            cols.append(u)
            ws.append(w)
    lv = np.stack([llc.compact(r) for r in lv]).astype(np.int32)
    nd = [int(r.max()) + 1 for r in lv] if nd is None else nd
    topo = synth.Topology(row_ptr, np.asarray(cols, np.int32), np.asarray(ws, np.int32),
                          np.asarray(free, np.int32).copy(), lv[0].copy(), np.full(nd[0], -1, np.int32))
    return topo, lv, nd


def grp(gid, level, hub=None, S=2, C=-1, pend=1, flags=STEP_EXCLUSIVE, fixed=-1, rflags=ROLE_EXCLUSIVE, demand=1):
    anchors = [] if hub is None else [(hub, 0, 8)]
    return (Group(gid=gid, roles=[(0, pend, demand, rflags)], pair=[[1]], anchors=anchors, flags=flags,
                  fixed_domain=fixed, level=level), [(S, C)])


def case(name, topo, lv, nd, gs, occ=None, **kw) -> Case:
    return Case(topo, [g for g, _ in gs], [r for _, r in gs], lv, nd,
                np.zeros((0, 3), np.int32) if occ is None else occ, name=name, **kw)


# ---------------------------------------------------------------- 1. list churn
def _churn_topo(n=32):
    """Zones (level 2) of 4 nodes, hostnames (level 1), level 0 one domain per node but D0 = {0, 12}; nodes 24.. are
    hubs (free 0).  Hub 24 -> 12 (E), 25 -> 0 (x) / 8 (y), 26 -> 2 (q), 27 -> 1 (z) / 4 (w)."""
    ids = np.arange(n)
    l0 = ids.copy()
    l0[12] = 0
    free = np.where(ids >= 24, 0, 4)
    edges = [(24, 12, 1000), (25, 0, 1000), (25, 8, 500), (26, 2, 1000), (27, 1, 1000), (27, 4, 500)]
    return graph(n, edges, free, [l0, ids, ids // 4])


def churn(kind: str) -> Case:
    """E (gid 1, level 0) reports D0 = {0, 12} from node 12.  H (gid 2) takes node 0 of zone 0 in round 1 and moves to
    node 8 in round 2 once it sees D0.  R (gid 3) wants node 1 of zone 0 and falls back to node 4 of zone 1.
      'pods'    H hostname-keyed: zone 0's pod list holds H's 2 pods in round 2 and is gone in round 3;
      'shrink'  plus Q (gid 3, hostname-keyed) on node 2: zone 0's pod list goes from 3 entries to 1 (R's own gid);
      'domain'  H zone-keyed, R hostname-keyed: the domain list of zone 0 (H's report) is gone in round 3."""
    topo, lv, nd = _churn_topo()
    E = grp(1, 0, hub=24, C=2)
    if kind == "domain":
        gs = [E, grp(2, 2, hub=25, C=1), grp(3, 1, hub=27)]
    else:
        gs = [E, grp(2, 1, hub=25)] + ([grp(3, 1, hub=26, S=1)] if kind == "shrink" else []) + [grp(3, 2, hub=27, C=1)]
    return case(f"churn_{kind}", topo, lv, nd, gs, rounds=3, tags={f"churn_{kind}"},
                extra=dict(zone=(2, 0), reader=len(gs) - 1, mover=1))


def churn_facts(c: Case, rs: Optional[List[Round]] = None) -> dict:
    """The list at extra['zone'] in rounds 2 and 3, and the reader's round-3 choice against the round-3 claims with the
    mover's round-2 claims put back (as if the list had kept its old entries)."""
    rs = replay(c) if rs is None else rs
    k, g, m = c.extra["zone"], c.extra["reader"], c.extra["mover"]
    lists = (lambda r: r.dom_lists) if c.name == "churn_domain" else (lambda r: r.pod_lists)
    stale = list(rs[1].claims[:g])        # what round 3 read, with the mover's claims that round 2 read
    stale[m] = rs[0].claims[m]
    off = pod_offsets(c)
    now = rs[2].assign[off[g]:off[g + 1]]
    return dict(rounds=len(rs), before=lists(rs[1]).get(k, 0), after=lists(rs[2]).get(k, 0),
                reader_moves=rs[1].assign[off[g]] != now[0],
                stale_differs=not np.array_equal(rerun(c, g, stale)[0], now),
                reader_in_zone=int(c.lv[2][now[0]]) == k[1] if now[0] >= 0 else False)


# ---------------------------------------------------------------- 2. claims only the final lists carry
def final_lists() -> Case:
    """A (gid 1, zone-keyed) places in zone 0; B (gid 2, level 0, last) takes node 1 of zone 0 in round 1, sees A's
    zone in round 2 and moves to node 12, still reporting D0 = {1, 12}.  The last round read B's round-1 pods (zone 0's
    pod list); the final lists carry its node 12 and D0, which alone take node 1 from A's alternates."""
    n = 32
    ids = np.arange(n)
    l0 = ids.copy()
    l0[12] = 1
    free = np.where(ids >= 24, 0, 4)
    edges = [(24, 0, 1000), (24, 2, 900), (24, 3, 800), (25, 1, 1000), (25, 12, 500)]
    topo, lv, nd = graph(n, edges, free, [l0, ids, ids // 4])
    gs = [grp(1, 2, hub=24, pend=2), grp(2, 0, hub=25)]
    return case("final_lists", topo, lv, nd, gs, tags={"final_lists"})


def final_lists_facts(c: Case, rs: Optional[List[Round]] = None) -> dict:
    rs = replay(c) if rs is None else rs
    before = rs[-2].claims if len(rs) > 1 else [NONE] * len(c.groups)   # what the last round's lists were built from
    _, last, pods = claims_view(c, before)
    exp = c.expected_ranked(8)
    stale = c.expected_ranked(8, claims=(last, pods))
    a_alts = exp[4][:pod_offsets(c)[1]]
    return dict(rounds=len(rs), last_changed=key(rs[-1]) != key(rs[-2]) if len(rs) > 1 else True,
                alt_differs=not np.array_equal(exp[4], stale[4]), node1_removed=1 not in a_alts.ravel().tolist(),
                a_zone=int(c.lv[2][exp[0][0]]))


# ---------------------------------------------------------------- 3. chains of exactly G rounds
def _chain_levels(kind: str, G: int) -> List[int]:
    if kind == "P":
        return [2 if i % 2 == 0 else 1 for i in range(G)]
    if kind == "K":
        return [3 if i % 2 == 0 else 6 for i in range(G)]
    return [i % 8 for i in range(G)]


def chain(G: int, kind: str) -> Case:
    """Hub h_i = 3i (free 0), a_i = 3i + 1 (edge 1000), b_i = 3i + 2 (edge 100); group i (gid 1000 + i) holds 2 replicas
    of 2 pods, co-located at level 0 on even i.  Group i takes b_i exactly when group i - 1 holds a_{i-1} and that
    claim reaches a_i: 'P' a_{i-1}, a_i share a domain at group i's level only (the pods' list), 'K' at group i - 1's
    level only (its report), 'mix' levels i % 8, P links into even i, K into odd i."""
    n = 3 * G
    levels = _chain_levels(kind, G)
    n_lv = 8 if kind == "mix" else max(levels) + 1
    parent = [np.arange(n, dtype=np.int64) for _ in range(n_lv)]

    def join(L, x, y):
        p = parent[L]
        p[p == p[y]] = p[x]
    for i in range(1, G):
        link = kind if kind != "mix" else ("P" if i % 2 == 0 else "K")
        join(levels[i] if link == "P" else levels[i - 1], 3 * i - 2, 3 * i + 1)
    free = np.full(n, 4, np.int32)
    free[0::3] = 0
    edges = [(3 * i, 3 * i + 1, 1000) for i in range(G)] + [(3 * i, 3 * i + 2, 100) for i in range(G)]
    topo, lv, nd = graph(n, edges, free, parent)
    gs = [grp(1000 + i, levels[i], hub=3 * i, pend=2, C=0 if i % 2 == 0 else -1) for i in range(G)]
    return case(f"chain_{kind}{G}", topo, lv, nd, gs, rounds=G, tags={"chain", f"chain_{kind}"},
                extra=dict(a=[3 * i + 1 for i in range(G)], b=[3 * i + 2 for i in range(G)]))


def chain_facts(c: Case, replay_rounds: bool = True) -> dict:
    G = len(c.groups)
    a, s, d = c.expected()
    want = [c.extra["a"][i] if i % 2 == 0 else c.extra["b"][i] for i in range(G)]
    f = dict(alternates=a.reshape(G, 4).tolist() == [[x] * 4 for x in want], all_placed=bool((s == 0).all()),
             lmask=lmask(c.groups))
    for terms in (("K",), ("P",)):
        f["without_" + "KP"[terms == ("K",)]] = not np.array_equal(c.expected(terms=terms)[0], a)
    if replay_rounds:
        rs = replay(c)
        f["rounds"] = len(rs)
        f["replay_final"] = key(rs[-1]) == (a.tolist(), s.tolist(), d.tolist())
    return f


CHAINS = [(8, "P"), (32, "P"), (8, "K"), (32, "K"), (8, "mix"), (32, "mix")]
REFRESH_CHAIN = (100, "mix")


# ---------------------------------------------------------------- 4. all eight levels, sparse masks
def levels(seed: int, n: int, excl: Sequence[int], other: Sequence[int], n_groups: int = 24,
           pairs: Sequence[tuple] = ()) -> Case:
    """lw_commit_gen's groups over partitions47: exclusive groups at `excl` in turn, the others at `other`; C drawn
    from -1..7; `pairs`: (exclusive level, C) forced on the first exclusive groups; records at levels 1..7."""
    f = lg.fleet(seed, n, n_groups=n_groups, scarce=True, levels=True, S_max=4)
    topo = f.topo
    lv, nd = llc.partitions47(topo, seed, "random")
    rng = np.random.default_rng(seed + 3)
    groups, rps, ke, ko = [], [], 0, 0
    for g, rp in zip(f.groups, f.rp):
        ex = bool(g.flags & STEP_EXCLUSIVE)
        C = [int(rng.choice([-1, 0, 1, 2, 3, 4, 5, 6, 7])) for _ in rp]
        if ex:
            L = excl[ke % len(excl)]
            if ke < len(pairs):
                L, C = pairs[ke][0], [pairs[ke][1]] * len(rp)
            ke += 1
        else:
            L = other[ko % len(other)]
            ko += 1
        fixed = g.fixed_domain
        if fixed >= 0:
            fixed = int(rng.integers(0, nd[L])) if ex else -1
        groups.append(dataclasses.replace(g, level=int(L), fixed_domain=fixed))
        rps.append([(S, c) for (S, _), c in zip(rp, C)])
    gids = sorted({g.gid for g in groups})
    occ = llc.keyed_records(np.random.default_rng(seed + 5), n, gids[:3] + [999], max(1, n // 40),
                            [1, 2, 3, 4, 5, 6, 7])
    m = "".join(map(str, excl))
    return Case(topo, groups, rps, lv, nd, occ, name=f"levels_{m}_{n}", tags={f"lmask_{m}"},
                extra=dict(excl=tuple(excl), other=tuple(other), pairs=tuple(pairs)))


def levels_cases() -> List[Case]:
    every = tuple(range(8))
    return [levels(71, 517, every, (1, 2, 3, 4, 5, 6, 7), 32, pairs=((3, 7), (7, 3))),
            levels(72, 1030, every, (1, 4, 6), 28, pairs=((7, 3), (3, 7))),
            sparse((3, 7), (1, 2, 4, 5, 6)), sparse((0, 2, 5), (1, 3, 4, 6, 7))]


def levels_facts(c: Case) -> dict:
    gr = c.groups
    ex = {g.level for g in gr if g.flags & STEP_EXCLUSIVE}
    ot = {g.level for g in gr if not g.flags & STEP_EXCLUSIVE}
    pairs = {(g.level, C) for g, rp in zip(gr, c.rp) if g.flags & STEP_EXCLUSIVE for _, C in rp}
    a, s, d = c.expected()
    return dict(lmask=lmask(gr), excl=ex, other=ot, pairs=pairs, placed=int((s == 0).sum()),
                multi_pod=any(S >= 2 for rp in c.rp for S, _ in rp),
                without_K=not np.array_equal(c.expected(terms=("P",))[0], a),
                without_P=not np.array_equal(c.expected(terms=("K",))[0], a))


# ---------------------------------------------------------------- claimers and the readers they move
def claims_and_readers(name: str, specs, others=(), tags=()) -> Case:
    """One claim per spec (kind, level L, end, reader level, claimer level) and a reader it moves, on eight levels.
    Per spec five nodes: the reader's hub (free 0) with edges 1000 to t and 100 to f, the claimer's hub (free 0) with
    edge 1000 to c.  At level L, t and c form one domain, the first ('first'), the last ('last') or an inner one
    ('mid') of the level; every other domain of every level is a single node.  The claimer (gid 2000 + k) is
      'report' exclusive at L, fixed to that domain, its one pod on c;   'idle' the same with nothing pending;
      'pods'   exclusive at the claimer level (!= L), its one pod on c.
    All claimers come first.  Reader k (gid 4000 + k, 2 replicas of 2 pods) is exclusive at the reader level: t is its
    best node, and the claim keeps it out, through K for 'report' / 'idle' (reader level != L) and through P for 'pods'
    (reader level = L), so it lands on f.  `others`: a non-exclusive group per level with its own hub and node."""
    N = 5 * len(specs) + 2 * len(others)
    ids = np.arange(N, dtype=np.int64)
    rows = [ids + 1 for _ in range(8)]
    free = np.full(N, 4, np.int32)
    edges = []
    for k, (kind, L, end, rl, cl) in enumerate(specs):
        hr, t, f, hc, cn = 5 * k + np.arange(5)
        free[[hr, hc]] = 0
        edges += [(hr, t, 1000), (hr, f, 100), (hc, cn, 1000)]
        rows[L] = rows[L].copy()
        rows[L][[t, cn]] = {"first": -1, "last": 10 * N, "mid": N + 1 + k}[end]
    base = 5 * len(specs)
    for j in range(len(others)):
        free[base + 2 * j] = 0
        edges.append((base + 2 * j, base + 2 * j + 1, 1000))
    topo, lv, nd = graph(N, edges, free, rows)
    claimers, readers, claims = [], [], []
    for k, (kind, L, end, rl, cl) in enumerate(specs):
        hr, t, f, hc, cn = 5 * k + np.arange(5)
        d = int(lv[L][cn])
        claims.append((L, d))
        if kind == "pods":
            claimers.append(grp(2000 + k, cl, hub=int(hc), S=1))
        else:
            claimers.append(grp(2000 + k, L, hub=int(hc), S=1, pend=0 if kind == "idle" else 1, fixed=d))
        readers.append(grp(4000 + k, rl, hub=int(hr), pend=2, C=-1 if k % 2 else (rl + 5) % 8))
    extra = [grp(6000 + j, L, hub=base + 2 * j, flags=0, C=(L + 1) % 8) for j, L in enumerate(others)]
    return case(name, topo, lv, nd, claimers + extra + readers, tags=set(tags),
                extra=dict(specs=list(specs), claims=claims, t=[5 * k + 1 for k in range(len(specs))],
                           f=[5 * k + 2 for k in range(len(specs))], first_reader=len(specs) + len(others)))


def moved_facts(c: Case) -> dict:
    """Per spec: the reader's pods all on f with the claim, all on t without the term the claim is read through; and
    whether the claimer holds its domain."""
    a, s, d = c.expected()
    off = pod_offsets(c)
    without = {"K": c.expected(terms=("P",))[0], "P": c.expected(terms=("K",))[0]}
    moved, held = [], []
    for k, (kind, L, end, rl, cl) in enumerate(c.extra["specs"]):
        g = c.extra["first_reader"] + k
        mine = slice(off[g], off[g + 1])
        wo = without["P" if kind == "pods" else "K"]
        moved.append(bool((a[mine] == c.extra["f"][k]).all() and (wo[mine] == c.extra["t"][k]).all()))
        L_, dm = c.extra["claims"][k]
        held.append(bool(d[k] == dm) if kind != "pods" else bool(a[off[k]] >= 0 and c.lv[L_, a[off[k]]] == dm))
    return dict(moved=moved, held=held)


def sparse(mask: Sequence[int], others: Sequence[int]) -> Case:
    """Exclusive groups only at the levels of `mask` (lmask's ranks differ from the levels), non-exclusive groups at
    `others`: for every ordered pair (x, y) of mask levels a report at x read from y and pods of y read at x, and one
    idle report at the last level read from the first."""
    specs = []
    for x in mask:
        for y in mask:
            if x != y:
                specs += [("report", x, "mid", y, -1), ("pods", x, "mid", x, y)]
    specs.append(("idle", mask[-1], "mid", mask[0], -1))
    m = "".join(map(str, mask))
    return _with(claims_and_readers(f"sparse_{m}", specs, others, tags={f"lmask_{m}"}), excl=tuple(mask),
                 other=tuple(others), pairs=())


def _with(c: Case, **kw) -> Case:
    c.extra.update(kw)
    return c


# ---------------------------------------------------------------- 5. level-offset edges
def offsets(kind: str) -> Case:
    """For every adjacent level pair (L, L + 1), claims on domain nd_L - 1 of L and domain 0 of L + 1, each by
    `kind` ('report', 'pods' or 'idle', see claims_and_readers); readers at L + 3 for reports, at L for pods (claimer
    at L + 1)."""
    specs = []
    for L in range(7):
        for lvl, end in ((L, "last"), (L + 1, "first")):
            specs.append((kind, lvl, end, lvl if kind == "pods" else (lvl + 3) % 8, (lvl + 1) % 8))
    return claims_and_readers(f"offsets_{kind}", specs, tags={f"offsets_{kind}"})


def offsets_facts(c: Case) -> dict:
    f = moved_facts(c)
    boundary = {(L, c.nd[L] - 1) for L in range(7)} | {(L + 1, 0) for L in range(7)}
    return dict(f, claimed_all=set(c.extra["claims"]) == boundary and all(f["held"]), levels=c.lv.shape[0],
                idle=sum(g.roles[0][1] == 0 for g in c.groups[:14]))


# ---------------------------------------------------------------- 6. long pod lists
def long_pods(kind: str, n: int = 4096, seed: int = 6) -> Case:
    """Zone level 2 of two zones: halves of the node range ('edge': they nest level 0's racks of 512) or a random half
    ('random': they do not).  64 hostname-keyed groups, one replica of 32 pods co-located per host, each fixed to its
    own node of zone 0 (free 32; the others 1): zone 0's pod list holds 2 048 entries of other gids.  Then 4 zone-keyed
    groups of 2 replicas of 2 pods (gangs on odd k)."""
    ids = np.arange(n, dtype=np.int64)
    topo = llc.plain_topology(n, ids // 512, free=1, tiers=2)
    rng = np.random.default_rng(seed)
    zone = (ids >= n // 2).astype(np.int64) if kind == "edge" else (rng.permutation(n) >= n // 2).astype(np.int64)
    topo.free[zone == 0] = 32
    lv = np.stack([topo.domain, ids, zone]).astype(np.int32)
    nd = [int(r.max()) + 1 for r in lv]
    hosts = rng.choice(np.flatnonzero(zone == 0), size=64, replace=False)
    gs = [grp(5000 + k, 1, S=32, C=1, fixed=int(hosts[k])) for k in range(64)]
    gs += [grp(5200 + k, 2, pend=2, C=1 if k % 2 else -1, flags=STEP_EXCLUSIVE | (STEP_GANG if k % 2 else 0))
           for k in range(4)]
    return case(f"long_{kind}", topo, lv, nd, gs, tags={"long_pods", f"long_{kind}"})


def long_pods_facts(c: Case) -> dict:
    a, s, d = c.expected()
    off = pod_offsets(c)
    in0 = sum(int((c.lv[2][a[off[k]:off[k + 1]]] == 0).sum()) for k in range(64) if s[k] != 2)
    nests = llc.nests(c.lv[0], c.lv[2])
    return dict(pods_in_zone0=in0, readers=[int(x) for x in d[-4:]], nests=nests,
                without_P=not np.array_equal(c.expected(terms=("K",))[0], a))


# ---------------------------------------------------------------- 7. opted-out roles
def opted_out() -> Case:
    """X (gid 1, hostname-keyed) places its participating role on node 12 and its opted-out role (2 replicas of 2 pods)
    on node 1 of zone 0; R (gid 2, zone-keyed) wants node 1 / zone 0: the opted-out pods carry no label, so R gets
    it."""
    n = 32
    ids = np.arange(n)
    free = np.where(ids >= 24, 0, 8)
    edges = [(24, 12, 1000), (26, 1, 1000), (25, 1, 1000), (25, 4, 500)]
    topo, lv, nd = graph(n, edges, free, [ids // 2, ids, ids // 4])
    X = Group(gid=1, roles=[(0, 1, 1, ROLE_EXCLUSIVE), (0, 2, 1, 0)], pair=[[1, 0], [0, 1]],
              anchors=[(24, 0, 8), (26, 1, 8)], flags=STEP_EXCLUSIVE, level=1)
    gs = [(X, [(2, -1), (2, 2)]), grp(2, 2, hub=25, C=1)]
    return case("opted_out", topo, lv, nd, gs, tags={"opted_out"})


def opted_out_facts(c: Case) -> dict:
    a, s, d = c.expected()
    rs = replay(c)
    fin = rs[-1].claims
    counted = list(fin)
    cap, rep, pods = fin[0]
    counted[0] = (cap, rep, sorted(pods + [int(x) for x in a[2:6]]))
    return dict(participating=a[:2].tolist(), opted_out=a[2:6].tolist(), reader=a[6:8].tolist(),
                counted_differs=not np.array_equal(rerun(c, 1, counted)[0], a[6:8]), rounds=len(rs))


# ---------------------------------------------------------------- 8. gang failure mid-chain at a level >= 1
def gang_mid_chain() -> Case:
    """E (gid 1) and F (gid 5, gang of 2 replicas of 2 pods of demand 2, fixed to zone 0: a failed run still holds
    the domain it would report) are zone-keyed and both want zone 0, the only zone with room for F.  Round 1 places
    both there; in round 2 F sees E's zone and fails.  R (gid 1, hostname-keyed)
    wants node 3 of zone 0: kept out by F's report in round 2 (the last reporter of zone 0), back in round 3."""
    n = 32
    ids = np.arange(n)
    free = np.where(ids < 4, 4, np.where(ids >= 24, 0, 1))
    edges = [(24, 0, 1000), (25, 1, 1000), (25, 2, 900), (26, 3, 1000), (26, 8, 500)]
    topo, lv, nd = graph(n, edges, free, [ids // 2, ids, ids // 4])
    gs = [grp(1, 2, hub=24, S=1), grp(5, 2, hub=25, pend=2, C=1, demand=2, flags=STEP_EXCLUSIVE | STEP_GANG, fixed=0),
          grp(1, 1, hub=26, S=1)]
    return case("gang_mid_chain", topo, lv, nd, gs, rounds=3, tags={"gang_mid_chain"})


def gang_mid_chain_facts(c: Case) -> dict:
    rs = replay(c)
    kept = list(rs[-1].claims)
    kept[1] = ({}, 0, [])                   # the failed gang's report of zone 0 kept
    return dict(rounds=len(rs), f_round1=int(rs[0].status[1]), f_final=int(rs[-1].status[1]),
                reader=[int(r.assign[-1]) for r in rs], f_claims_final=rs[-1].claims[1] == NONE,
                kept_report_differs=rerun(c, 2, kept)[0].tolist() != rs[-1].assign[-1:].tolist())


# ---------------------------------------------------------------- 9. gids
def gids() -> Case:
    """Gids 0 (level 1) and 2^31 - 1 (level 2, co-located per host); gid 77 at level 1 on node 9 (zone 2), then gid 77
    at level 2 anchored there: its own pod is in its P.  Gids 11 then 12 report zone 5 (fixed), and a later gid-11
    group fixed to node 21 of zone 5 is kept out by the last reporter."""
    n = 40
    ids = np.arange(n)
    free = np.where(ids >= 32, 0, 4)
    edges = [(32, 0, 1000), (33, 4, 1000), (34, 9, 1000), (35, 9, 1000), (35, 10, 900), (35, 13, 500)]
    topo, lv, nd = graph(n, edges, free, [ids // 2, ids, ids // 4])
    gs = [grp(0, 1, hub=32), grp(GID_MAX, 2, hub=33, pend=2, C=1), grp(77, 1, hub=34), grp(77, 2, hub=35, pend=2),
          grp(11, 2, S=1, fixed=5), grp(12, 2, S=1, fixed=5), grp(11, 1, S=1, fixed=21)]
    return case("gids", topo, lv, nd, gs, tags={"gids"})


def gids_facts(c: Case) -> dict:
    a, s, d = c.expected()
    off = pod_offsets(c)
    regid = c.replace(groups=[dataclasses.replace(g, gid=78) if k == 2 else g for k, g in enumerate(c.groups)])
    ra = regid.expected()[0]
    return dict(gid_ends={0, GID_MAX} <= {g.gid for g in c.groups},
                own_pods_zone=int(c.lv[2][a[off[3]]]), first77_zone=int(c.lv[2][a[off[2]]]),
                shared_gid_matters=not np.array_equal(ra[off[3]:off[4]], a[off[3]:off[4]]),
                reporters=[int(d[4]), int(d[5])], last_keeps_out=int(a[off[6]]),
                first_differs=not np.array_equal(c.expected(reporter="first")[0], a))


# ---------------------------------------------------------------- 10. mixed-level emit blocks
def emit_blocks(n: int = 1024, seed: int = 9, G: int = 40) -> Case:
    """One wave of G one-role groups (G >= 33 steps): exclusive levels 1, 2, 3, 5, 6, 7, 0 in turn between adjacent
    steps with a non-exclusive step every fifth, gids alternating among 7, all anchored on a few nodes so that each
    group's claims reach the next ones."""
    topo = synth.make_topology(n, seed=seed, tiers=2, max_free=4)
    topo.domain_owner[:] = -1
    topo.free = np.full(n, 2, np.int32)
    lv, nd = llc.partitions47(topo, seed, "random")
    rng = np.random.default_rng(seed)
    hot = rng.choice(n, 6, replace=False)
    order = [1, 2, 3, 5, 6, 7, 0]
    gs = []
    for k in range(G):
        ex = k % 5 != 4
        g, rp = grp(100 + k % 7, order[k % 7], S=2, C=[-1, 0, 2, 7][k % 4], pend=1 + k % 2,
                    flags=STEP_EXCLUSIVE if ex else 0)
        g.anchors = [(int(hot[k % 6]), 0, 16)]
        gs.append((g, rp))
    return case("emit_blocks", topo, lv, nd, gs, tags={"emit_blocks"})


def emit_blocks_facts(c: Case) -> dict:
    gr = c.groups
    adj = sum(1 for x, y in zip(gr, gr[1:]) if x.level != y.level and x.gid != y.gid)
    a, s, d = c.expected()
    waves = [len(X.waves) for X in lco.groups_of(c.blob(), c.role_pods())]
    return dict(steps=len(gr), one_wave=waves == [1] * len(gr),
                adjacent_mixed=adj, non_exclusive=sum(not g.flags & STEP_EXCLUSIVE for g in gr),
                without_K=not np.array_equal(c.expected(terms=("P",))[0], a),
                without_P=not np.array_equal(c.expected(terms=("K",))[0], a))


# ---------------------------------------------------------------- 11. ragged chunks
def ragged(n: int) -> Case:
    """N = 4 097 or 129: node n - 1 is the best (edge 1000 from hub 0, which has free 0); windows of 100 nodes (level
    2) straddle the 128- and 2 048-node chunk boundaries; groups at levels 1 and 2 claim across them."""
    ids = np.arange(n)
    free = np.where(ids == 0, 0, 2)
    edges = [(0, n - 1, 1000), (0, n - 2, 900)]
    for b in (128, 2048, 4096):
        if b < n - 2:
            edges += [(0, b - 1, 800), (0, b, 700)]
    topo, lv, nd = graph(n, edges, free, [ids // 64, ids, (ids + 36) // 100])
    gs = [grp(1, 1, hub=0, S=2), grp(2, 2, hub=0, S=2, C=1), grp(3, 2, hub=0, pend=2, C=-1),
          grp(1, 2, hub=0, S=1), grp(4, 1, hub=0, S=2, flags=STEP_EXCLUSIVE | STEP_GANG), grp(5, 0, hub=0, S=2, C=2)]
    return case(f"ragged_{n}", topo, lv, nd, gs, tags={"ragged"})


def ragged_facts(c: Case) -> dict:
    a, s, d = c.expected()
    n = c.topo.n
    straddle = [int(c.lv[2][b - 1]) == int(c.lv[2][b]) for b in (128, 2048, 4096) if b < n]
    return dict(first_last=int(a[0]), straddle=straddle, placed=int((s == 0).sum()))


# ---------------------------------------------------------------- 12. scale
def million(n: int = llc.FULL_N, G: int = 12) -> Case:
    """llc.derivation's seven levels and 610 000 records; G groups of distinct gids over all eight levels (exclusive
    at every level but 6 for G = 12), 2-pod replicas, gangs.  No group has anchors: all of them rank the nodes by the
    background order alone and race for its head, so each group's claims reach the groups after it (a short chain of
    claims, at the low node ids)."""
    dv = llc.derivation(n)
    gs = []
    for k in range(G):
        g, rp = grp(6000 + k % 40, k % 8, S=2, C=[-1, 1, 2, 3][k % 4], pend=1 + k % 3,
                    flags=STEP_EXCLUSIVE | (STEP_GANG if k % 5 == 4 else 0) if k % 6 else 0)
        gs.append((g, rp))
    return case(f"million_{n}", dv.topo, dv.lv, dv.nd, gs, occ=dv.occ, tags={"million"})


def bitmap_ceiling(n: int = 200 * 1024 * 8) -> Case:
    """Exactly the room bitmap's 1 638 400 nodes, three levels (hostname, racks of 16, level-0 eighths)."""
    topo = synth.make_topology(n, seed=31, tiers=2, max_free=2)
    topo.domain = (np.arange(n) // (n // 8)).astype(np.int32)
    topo.domain_owner = np.full(8, -1, np.int32)
    ids = np.arange(n)
    lv = np.stack([topo.domain, ids, ids // 16, ids // 4096]).astype(np.int32)
    nd = [8, n, n // 16, n // 4096]
    gs = [grp(1, 1, S=2), grp(2, 2, S=2, C=1, pend=2), grp(3, 3, S=2, C=2), grp(1, 0, S=2, C=3),
          grp(4, 2, S=1, flags=0)]
    gs[0][0].anchors = [(n - 1, 0, 4)]
    return case("bitmap_ceiling", topo, lv, nd, gs, tags={"bitmap_ceiling"})


# ---------------------------------------------------------------- 13. the exactness bound at a level
def exact(case_i: int):
    """test_gpu_lw_limits.EXACT_CASES[case_i] as a group exclusive at level 2 (racks of 16) whose real roles
    participate: (the case with `count` anchors, the count at the bound)."""
    import groups_gen as gg
    from test_gpu_lw_limits import EXACT_CASES, enumerated_bound, exact_group, free_topo
    pair, S, pend, gang = EXACT_CASES[case_i]
    n = 130
    topo = free_topo(n, 29, max_free=3)
    topo.free[np.random.default_rng(29).random(n) < 0.6] = 0
    roles, full = exact_group(pair, pend)
    B = enumerated_bound(roles[:-1], [r[:-1] for r in full[:-1]], list(S), gang)
    roles = [(r[0], r[1], r[2], ROLE_EXCLUSIVE) for r in roles[:-1]] + roles[-1:]
    row_w = gg.wsum_max(topo) + 8000
    c_at = ((1 << 24) + row_w - 1) // row_w - max(B)
    ids = np.arange(n)
    lv = np.stack([topo.domain, ids, ids // 16]).astype(np.int32)
    nd = [len(topo.domain_owner), n, (n + 15) // 16]

    def at(count: int) -> Case:
        g = Group(gid=1, roles=roles, pair=full, anchors=[(7, len(pend), count)],
                  flags=STEP_EXCLUSIVE | (STEP_GANG if gang else 0), level=2)
        return Case(topo, [g], [[(x, -1) for x in S] + [(1, -1)]], lv, nd, np.zeros((0, 3), np.int32),
                    name=f"exact{case_i}", tags={"exactness_at_level"})
    return at, c_at


# ---------------------------------------------------------------- the seed set and its coverage
def cases() -> List[Case]:
    return ([churn(k) for k in ("pods", "shrink", "domain")] + [final_lists()] + [chain(G, k) for G, k in CHAINS]
            + levels_cases() + [offsets(k) for k in ("report", "pods", "idle")]
            + [long_pods(k) for k in ("edge", "random")]
            + [opted_out(), gang_mid_chain(), gids(), emit_blocks(), ragged(4097), ragged(129)])


BULLETS = ("churn_pods", "churn_shrink", "churn_domain", "final_lists", "chain_P", "chain_K", "chain_mix",
           "lmask_ff", "colocate_7_excl_3", "colocate_3_excl_7", "sparse_37", "sparse_025", "offsets_report",
           "offsets_pods", "offsets_idle", "long_edge", "long_random", "opted_out", "gang_mid_chain", "gid_ends",
           "shared_gid_levels", "two_reporters", "emit_blocks", "ragged_4097", "ragged_129", "multi_pod",
           "colocation_off_level", "scale_million", "scale_bitmap_ceiling", "exactness_at_level")


def coverage(cs: List[Case]) -> Dict[str, bool]:
    """Which bullets the cases reach, each judged by the facts its case was built for (a case that stops churning,
    moving its readers or needing its term stops covering its bullet)."""
    c = dict.fromkeys(BULLETS, False)
    for x in cs:
        gr = x.groups
        m = lmask(gr)
        pairs = {(g.level, C) for g, rp in zip(gr, x.rp) if g.flags & STEP_EXCLUSIVE for _, C in rp}
        c["colocate_7_excl_3"] |= (3, 7) in pairs
        c["colocate_3_excl_7"] |= (7, 3) in pairs
        c["multi_pod"] |= any(S >= 2 for rp in x.rp for S, _ in rp)
        c["colocation_off_level"] |= any(C >= 0 and C != L for L, C in pairs)
        n = x.name
        if n.startswith("churn_"):
            f = churn_facts(x)
            c[n] |= f["rounds"] == 3 and f["stale_differs"] and f["before"] > f["after"]
        elif n == "final_lists":
            f = final_lists_facts(x)
            c[n] |= f["alt_differs"] and f["last_changed"]
        elif n.startswith("chain_") and len(gr) == 8:
            f = chain_facts(x)
            need = {"P": f["without_P"], "K": f["without_K"], "mix": f["without_K"] and m == 0xFF}
            c["chain_" + n[6:-1]] |= f["rounds"] == 8 and need[n[6:-1]]
        elif n.startswith("levels_"):
            f = levels_facts(x)
            c["lmask_ff"] |= m == 0xFF and (f["without_K"] or f["without_P"])
        elif n.startswith("sparse_") or n.startswith("offsets_"):
            f = moved_facts(x)
            c[n] |= all(f["moved"]) and all(f["held"])
        elif n.startswith("long_"):
            f = long_pods_facts(x)
            c[n] |= f["pods_in_zone0"] >= 2048 and f["without_P"]
        elif n == "opted_out":
            c[n] |= opted_out_facts(x)["counted_differs"]
        elif n == "gang_mid_chain":
            f = gang_mid_chain_facts(x)
            c[n] |= f["f_round1"] == 0 and f["f_final"] == 2 and f["kept_report_differs"]
        elif n == "gids":
            f = gids_facts(x)
            c["gid_ends"] |= f["gid_ends"]
            c["shared_gid_levels"] |= f["shared_gid_matters"]
            c["two_reporters"] |= f["reporters"][0] == f["reporters"][1] >= 0 and f["first_differs"]
        elif n == "emit_blocks":
            f = emit_blocks_facts(x)
            c[n] |= f["one_wave"] and f["steps"] >= 33 and f["adjacent_mixed"] >= 32
        elif n.startswith("ragged_"):
            f = ragged_facts(x)
            c[n] |= f["first_last"] == x.topo.n - 1 and all(f["straddle"])
    return c


def scale_and_bound_coverage() -> Dict[str, bool]:
    """The GPU-only bullets, judged on their builders: sizes, levels and the level of the bounded group."""
    mil, bm = million(), bitmap_ceiling()
    at, c_at = exact(0)
    ex = at(c_at)
    return dict(scale_million=mil.topo.n == (1 << 20) + 1 and mil.lv.shape[0] == 8
                and bin(lmask(mil.groups)).count("1") >= 7,
                scale_bitmap_ceiling=bm.topo.n == 200 * 1024 * 8 and bm.lv.shape[0] == 4,
                exactness_at_level=ex.groups[0].level >= 1 and bool(ex.groups[0].flags & STEP_EXCLUSIVE))
