"""Designed fleets whose dense matrix passes 2^31 elements, with the boundary inside a row (test infrastructure).

Every kernel that touches the dense matrix forms a row's address as (size_t)row * slab_stride.  At N = 300 000 a fleet
of 900 groups, each one wave of 8 roles x 1 replica, has 7 200 role rows: about 8.1 GiB of floats, so the element
index 2^31 falls inside row r* = 2^31 // slab_stride, at node n* = 2^31 % slab_stride.  slab_stride depends on the
chunk configuration (compute_slab):
  - the default chunk: slab_stride = 147 x 2048 = 301 056, r* = 7 133, n* = 51 200 (a chunk boundary);
  - chunk_nodes = 1920: slab_stride = 157 x 1920 = 301 440, r* = 7 124, n* = 25 088 = 13 x 1920 + 128, inside a
    CTA's chunk.
Rows are in group order, so groups 889-892 hold both straddling rows and one fleet serves both configurations.

Most groups are identical non-exclusive fillers: under snapshot semantics (DESIGN.md §3.7) each copy gets the same
placements and the same rows, so one oracle run covers all of them.  The distinct groups are group 0 (where a row
offset wrapped to 31 bits would land), the straddle groups 889-892 and the last group.  The straddle groups are
exclusive, with anchors whose closed neighbourhoods hold nodes on both sides of each n*, and anchors that put the
best nodes of every role above n*.

The fleets: `groups_fleet` (stage_groups / place_groups[_ranked], and leader-worker with `lw_role_pods`),
`steps_fleet` (stage / score_assign: 900 steps of 8 roles, the straddling steps anchored on a hub whose neighbourhood
is past shared memory, plus a consumed record just above n*) and `rerun_fleet` (two-wave fillers whose first wave
leaves a replica unplaced, so every group goes through the host-driven loop and its kept rows pass 2^31 floats).
Each has a `*_pre` check that proves, from plan_steps row numbers, N and the oracle, that the fleet still reaches its
edge."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Sequence

import numpy as np

import steps_gen as sg
import topo_gen as tg
from rbg_b200 import synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, STEP_GANG, Group, GroupsBuilder, Step

N = 300_000
G = 900
Q = 8                                  # roles per group, one replica each: one wave of 8 role rows
TWO31 = 1 << 31
CHUNKS = (0, 1920)                     # chunk_nodes of the two configurations (0: the default chunk)
STRADDLE = (889, 890, 891, 892)
SEED = 21
FILLER_GID0, DISTINCT_GID0 = 10_000, 20_000


def round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


def slab_stride(n: int, chunk_nodes: int = 0) -> int:
    """compute_slab at world 1: floats per dense row."""
    tcfg = min(2048, max(128, round_up(chunk_nodes if chunk_nodes > 0 else 2048, 128)))
    lc = max(1, (n + tcfg - 1) // tcfg)
    chunk = min(2048, max(128, round_up((n + lc - 1) // lc, 128)))
    return round_up(max(1, lc * chunk), 32)


def straddle(n: int, chunk_nodes: int = 0, at: int = TWO31):
    """(r*, n*): the row that holds element index `at` and the node where it falls."""
    s = slab_stride(n, chunk_nodes)
    return at // s, at % s


def pivots(n: int = N) -> List[int]:
    """The n* of every chunk configuration at N = n (at a scaled-down n: two nodes standing in for them)."""
    if n == N:
        return [straddle(n, c)[1] for c in CHUNKS]
    return [n // 3, n // 2 + 4]


def topology(n: int = N, piv=None) -> synth.Topology:
    """A two-tier synth cluster (its NVLink cliques and sampled peers never cross a multiple of 2048) with bridges:
    four edges of weight 10 across every pivot, so anchors there reach both sides.  Domains of 8 nodes, 20 % of them
    owned by foreign gids, free 0-4."""
    base = synth.make_topology(n, seed=SEED, tiers=2, max_free=4)
    u, v, w = tg.edges_of(base)
    bu, bv = [], []
    for pv in (pivots(n) if piv is None else piv):
        bu += [pv - 1 - i for i in range(4)]
        bv += [pv + 3 + 5 * i for i in range(4)]
    return tg.from_edges(n, np.concatenate([u, bu]), np.concatenate([v, bv]), np.concatenate([w, [10] * len(bu)]),
                         base.free, owned_frac=0.2, seed=SEED)


def closed_nbhd(topo, a: int) -> np.ndarray:
    return np.concatenate([[a], topo.col_idx[topo.row_ptr[a]:topo.row_ptr[a + 1]]])


def spanning_anchor(topo, pivot: int) -> int:
    """The node nearest below `pivot` whose closed neighbourhood holds nodes on both sides of it."""
    for a in range(pivot - 1, max(pivot - 4096, -1), -1):
        nb = closed_nbhd(topo, a)
        if (nb >= pivot).any() and (nb < pivot).any():
            return a
    raise AssertionError(f"no anchor spans node {pivot}")


def open_node_above(topo, pivot: int) -> int:
    """The first node >= pivot with free >= 2 whose domain no foreign gid owns."""
    own = topo.domain_owner[topo.domain]
    for m in range(pivot, min(pivot + 4096, topo.n)):
        if topo.free[m] >= 2 and own[m] == -1:
            return m
    raise AssertionError(f"no open node above {pivot}")


def _pair(rng, q: int = Q) -> List[List[int]]:
    p = rng.integers(0, 3, size=(q, q))
    np.fill_diagonal(p, 0)
    return p.tolist()


def _roles(level: int = 0, demand: int = 1, q: int = Q, flags: int = ROLE_EXCLUSIVE) -> List[tuple]:
    return [(level, 1, demand, flags) for _ in range(q)]


def filler(gid: int, n: int) -> Group:
    p = np.ones((Q, Q), dtype=np.int64)
    np.fill_diagonal(p, 0)
    return Group(gid=gid, roles=_roles(), pair=p.tolist(), anchors=[(n // 7, 0, 1), (5 * n // 7, 3, 2)])


HEAVY_ROLE, HEAVY_NODES = Q - 2, 2000


def straddle_group(topo, gid: int, k: int, piv: Sequence[int], heavy: bool = False) -> Group:
    """Exclusive, every role participating.  For every pivot: an anchor of role k % Q whose neighbourhood spans it,
    and three pods of role Q - 1 on an open node above it, which every other role pairs with at weight 2, so the best
    nodes of the straddling rows lie above n*.  heavy: HEAVY_NODES more pods of HEAVY_ROLE (pair column 0) on
    distinct nodes, so the group's patched nodes fit neither k_plan_group's nor the fast selection's shared memory
    (the plan runs one launch per wave through k_select_assign's global candidate list)."""
    rng = np.random.default_rng(100 + k)
    pair = np.asarray(_pair(rng))
    pair[:, Q - 1] = 2
    pair[Q - 1, Q - 1] = 0
    anchors = []
    for pv in piv:
        anchors.append((spanning_anchor(topo, pv), k % Q, 1))
        anchors.append((open_node_above(topo, pv + 4 * k), Q - 1, 3))
    if heavy:
        pair[:, HEAVY_ROLE] = 0
        nodes = np.random.default_rng(k).choice(topo.n, size=HEAVY_NODES, replace=False)
        anchors += [(int(x), HEAVY_ROLE, 1) for x in nodes]
    return Group(gid=gid, roles=_roles(), pair=pair.tolist(), anchors=anchors, flags=STEP_EXCLUSIVE)


def distinct_group(topo, gid: int, kind: str, n: int) -> Group:
    rng = np.random.default_rng({"first": 1, "last": 2}[kind])
    anchors = [(int(rng.integers(0, n)), int(rng.integers(0, Q)), int(rng.integers(1, 3))) for _ in range(4)]
    if kind == "first":    # exclusive, demand 2, a different pair matrix: rows unlike any filler's
        return Group(gid=gid, roles=_roles(demand=2), pair=_pair(rng), anchors=anchors, flags=STEP_EXCLUSIVE)
    return Group(gid=gid, roles=_roles(), pair=_pair(rng), anchors=anchors, flags=STEP_GANG)


@dataclass
class Fleet:
    topo: synth.Topology
    groups: List[Group]
    blob: np.ndarray
    rep: List[int]            # rep[g]: the group whose oracle run stands for group g (itself, or the first filler)
    distinct: List[int]       # the groups the oracle runs (every distinct group and the representative filler)
    pivots: List[int]
    kinds: Dict[int, str]     # the distinct groups: "first", "straddle" or "last"


def _build(groups) -> np.ndarray:
    gb = GroupsBuilder()
    for g in groups:
        gb.add(g)
    return gb.build()


def _positions(n_groups: int, straddles: Sequence[int]) -> Dict[int, str]:
    pos = {0: "first", n_groups - 1: "last"}
    for g in straddles:
        pos[g] = "straddle"
    return pos


def _fleet(topo, groups, kinds: Dict[int, str], piv) -> Fleet:
    first_filler = next(g for g in range(len(groups)) if g not in kinds)
    rep = [g if g in kinds else first_filler for g in range(len(groups))]
    return Fleet(topo, groups, _build(groups), rep, sorted(set(kinds) | {first_filler}), list(piv), dict(kinds))


def groups_fleet(n: int = N, n_groups: int = G, straddles: Sequence[int] = STRADDLE, topo=None, piv=None,
                 heavy: Sequence[int] = ()) -> Fleet:
    """The GROUPS fleet: fillers, group 0, the straddle groups and the last group; piv: the n* to straddle (default
    pivots(n)); heavy: straddle groups whose patched nodes are past shared memory."""
    piv = pivots(n) if piv is None else piv
    topo = topology(n, piv) if topo is None else topo
    kinds = _positions(n_groups, straddles)
    groups = []
    for g in range(n_groups):
        kind = kinds.get(g)
        if kind is None:
            groups.append(filler(FILLER_GID0 + g, n))
        elif kind == "straddle":
            groups.append(straddle_group(topo, DISTINCT_GID0 + g, g, piv, heavy=g in heavy))
        else:
            groups.append(distinct_group(topo, DISTINCT_GID0 + g, kind, n))
    return _fleet(topo, groups, kinds, piv)


def lw_role_pods(fleet: Fleet) -> np.ndarray:
    """(S, C) per role: fillers (1, -1); the straddle groups cycle S over 1, 2, 4 and C over -1, 0, 1 (at most 32 pods
    per wave: 8 roles x 4); group 0 and the last group (2, 0) and (1, 1)."""
    out = []
    for g in range(len(fleet.groups)):
        kind = fleet.kinds.get(g)
        for r in range(Q):
            if kind is None:
                out.append((1, -1))
            elif kind == "first":
                out.append((2, 0))
            elif kind == "last":
                out.append((1, 1))
            else:
                out.append(((1, 2, 4)[(r + g) % 3], (-1, 0, 1)[(r + 2 * g) % 3]))
    return np.asarray(out, dtype=np.int32)


def lw_levels(topo) -> List[np.ndarray]:
    """Co-location partitions: level 0 = the snapshot's domains, level 1 = four of them together."""
    return [np.asarray(topo.domain, np.int32), np.asarray(topo.domain // 4, np.int32)]


def lw_topology(topo) -> synth.Topology:
    """The snapshot without owners: co-location levels put the context in occupancy mode, where owners come from pods."""
    return synth.Topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain,
                          np.full(len(topo.domain_owner), -1, np.int32))


# ---- re-run fleet: every group through the host-driven loop

def rerun_group(topo, gid: int, k: int, kind, n: int, piv) -> Group:
    """Two waves, non-gang: 8 roles in level 0, then one role in level 1.  Role 0 asks more than any node has, so the
    first wave leaves a replica unplaced and the plan hands the group to the host-driven loop.  That loop keeps the
    8 rows of every group's first wave, then the second wave's rows from kept row 8 x G on: past 2^31 floats."""
    big = int(topo.free.max()) + 1
    q = Q + 1
    roles = [(0, 1, big, ROLE_EXCLUSIVE)] + [(0, 1, 1, ROLE_EXCLUSIVE)] * (Q - 1) + [(1, 1, 1, ROLE_EXCLUSIVE)]
    p = np.ones((q, q), dtype=np.int64)
    np.fill_diagonal(p, 0)
    anchors = [(n // 7, 1, 1), (5 * n // 7, 5, 2)]
    flags = 0
    if kind == "straddle":
        rng = np.random.default_rng(300 + k)
        p = np.asarray(_pair(rng, q))
        p[:, 3] = 2
        p[3, 3] = 0
        anchors = [a for pv in piv for a in ((spanning_anchor(topo, pv), k % Q, 1), (open_node_above(topo, pv + 4 * k), 3, 3))]
        flags = STEP_EXCLUSIVE
    elif kind == "first":
        rng = np.random.default_rng(7)
        p = np.asarray(_pair(rng, q))
        anchors = [(int(rng.integers(0, n)), int(rng.integers(0, q)), 1) for _ in range(3)]
        flags = STEP_EXCLUSIVE
    elif kind == "last":
        anchors = [(n - 1, 2, 1), (n // 2, Q, 1)]
    return Group(gid=gid, roles=roles, pair=p.tolist(), anchors=anchors, flags=flags)


def rerun_fleet(n: int = N, n_groups: int = G, straddles: Sequence[int] = STRADDLE, topo=None) -> Fleet:
    piv = pivots(n)
    topo = topology(n, piv) if topo is None else topo
    kinds = _positions(n_groups, straddles)
    groups = [rerun_group(topo, (DISTINCT_GID0 if g in kinds else FILLER_GID0) + g, g, kinds.get(g), n, piv)
              for g in range(n_groups)]
    return _fleet(topo, groups, kinds, piv)


# ---- step batches

def steps_topology(n: int = N):
    """steps_gen's cluster: a hub linked to a quarter of the nodes, full nodes, owned domains."""
    topo, hubs, _ = sg.topology(SEED, n)
    return topo, hubs[0]


@dataclass
class StepFleet:
    topo: synth.Topology
    steps: List[Step]
    blob: np.ndarray
    rep: List[int]
    distinct: List[int]
    hub: int
    hub_steps: List[int]
    pivots: List[int]


def _light_node_near(topo, x: int, deg_max: int = 40) -> int:
    deg = np.diff(topo.row_ptr)
    for m in range(x, topo.n):
        if 0 < deg[m] < deg_max:
            return m
    raise AssertionError(x)


def steps_fleet(n: int = N, n_steps: int = G, straddles: Sequence[int] = STRADDLE, topo_hub=None) -> StepFleet:
    """900 steps of 8 roles x 1 replica (count, demand, need, flags).  The steps holding r* of either chunk
    configuration (890 and 891 at full size) also anchor on the hub with a pair column of weight 0 (the exactness
    bound holds whatever the hub's weight), so their patched set is past shared memory and the rows are corrected and
    read back through k_select_assign's global candidate list."""
    topo, hub = steps_topology(n) if topo_hub is None else topo_hub
    piv = pivots(n)
    limit = sg.amax_limit(topo)
    kinds = _positions(n_steps, straddles)
    hub_steps = sorted({straddle(n, c)[0] // Q for c in CHUNKS}) if n == N else [straddles[1], straddles[2]]
    a_lo, a_hi = _light_node_near(topo, n // 7), _light_node_near(topo, 5 * n // 7)
    steps = []
    for s in range(n_steps):
        kind = kinds.get(s)
        if kind is None:
            pair = np.ones((Q, Q), dtype=np.int64)
            np.fill_diagonal(pair, 0)
            st = Step(gid=FILLER_GID0 + s, roles=[(1, 1, 2, ROLE_EXCLUSIVE)] * Q, pair=pair.tolist(),
                      anchors=[(a_lo, 0, 1), (a_hi, 3, 1)], consumed=[(a_hi, 1)])
        else:
            rng = np.random.default_rng(500 + s)
            pair = rng.integers(0, 3, size=(Q, Q + 1))
            pair[:, Q] = 0
            anchors = [(int(_light_node_near(topo, int(rng.integers(0, n // 2)))), int(rng.integers(0, Q)), 1)
                       for _ in range(3)]
            consumed = []
            if kind == "straddle":
                for pv in piv:
                    anchors.append((spanning_anchor(topo, pv), s % Q, 1))
                    consumed.append((pv + s % 4, 1))                       # a consumed record just above n*
            if s in hub_steps:
                anchors.append((hub, Q, 1))
                consumed.append((hub, 1))
            demand = 2 if kind == "first" else 1
            st = Step(gid=DISTINCT_GID0 + s, roles=[(1, demand, 2, ROLE_EXCLUSIVE)] * Q, pair=pair.tolist(),
                      anchors=anchors, consumed=consumed,
                      flags=STEP_EXCLUSIVE if kind in ("straddle", "first") else (STEP_GANG if kind == "last" else 0))
            sg._lower_to_bound(st, limit)
            st.roles = [tuple(r) for r in st.roles]
        steps.append(st)
    first_filler = next(s for s in range(n_steps) if s not in kinds)
    rep = [s if s in kinds else first_filler for s in range(n_steps)]
    return StepFleet(topo, steps, sg.build(steps), rep, sorted(set(kinds) | {first_filler}), hub, hub_steps, piv)


def step_blob(fleet: StepFleet, s: int) -> np.ndarray:
    """A blob of step s alone (the oracle run that stands for every step with rep == s)."""
    return sg.build([fleet.steps[s]])


# ---- preconditions (no GPU)

def layout_pre(n: int = N, rows: int = G * Q) -> None:
    """Both chunk configurations: the straddling row is inside the matrix, 2^31 falls inside it with at least one
    float4 group of nodes on each side, and the matrix is below the 2^31 element count only without that row."""
    for c in CHUNKS:
        s = slab_stride(n, c)
        r, nstar = straddle(n, c)
        assert r * s + nstar == TWO31 and r < rows, (c, r, rows)
        assert 4 <= nstar <= n - 4 and nstar % 4 == 0, (c, nstar)
        assert rows * s > TWO31 and (rows - 1) * s < 2 * TWO31, (c, rows)
    if n == N:   # the default chunk straddles at a chunk boundary, chunk_nodes = 1920 inside a CTA's chunk
        assert straddle(n, 0) == (7133, 51_200) and straddle(n, 0)[1] % 2048 == 0
        assert straddle(n, 1920) == (7124, 25_088) and straddle(n, 1920)[1] % 1920 != 0


def plan_pre(fleet: Fleet) -> Dict[int, tuple]:
    """From rbgtopo_plan_describe: every group is one wave whose rows are 8g .. 8g + 7, and the straddling row of each
    configuration is a row of a straddle group.  Returns {chunk_nodes: (r*, n*, group, role)}."""
    from gpu_util import plan_rows
    rows = plan_rows(fleet.blob, fleet.topo)
    assert sorted(rows) == [(g, 0) for g in range(len(fleet.groups))], "every group one wave"
    assert all(rows[(g, 0)] == Q * g for g in range(len(fleet.groups)))
    out = {}
    for c in CHUNKS:
        r, nstar = straddle(fleet.topo.n, c)
        g, p = divmod(r, Q)
        assert g in STRADDLE, (c, r, g)
        out[c] = (r, nstar, g, p)
    return out


def anchors_pre(fleet: Fleet) -> None:
    """Every straddle group has, for each n*, an anchor whose closed neighbourhood spans it and anchor nodes above it."""
    for g in STRADDLE:
        grp = fleet.groups[g]
        for pv in fleet.pivots:
            spans = [a for a, _, _ in grp.anchors
                     if (closed_nbhd(fleet.topo, a) >= pv).any() and (closed_nbhd(fleet.topo, a) < pv).any()]
            assert spans, (g, pv)
            assert any(a >= pv for a, _, _ in grp.anchors), (g, pv)
        assert grp.flags & STEP_EXCLUSIVE and all(r[3] & ROLE_EXCLUSIVE for r in grp.roles), g


def wrap_alias_pre(rows_of, n: int = N) -> None:
    """A row offset wrapped to 31 bits moves the tail [n*, N) of the straddling row onto row 0's nodes [0, N - n*):
    group 0's row 0 must differ there from the straddling row's tail, or the wrap would store identical bits.
    rows_of(g) -> the oracle's [8][N] rows of group g."""
    r0 = rows_of(0)[0].view(np.uint32)
    for c in CHUNKS:
        r, nstar = straddle(n, c)
        tail = rows_of(r // Q)[r % Q].view(np.uint32)[nstar:]
        assert (r0[:len(tail)] != tail).sum() > len(tail) // 2, c


def best_above_pre(rows_of, fleet: Fleet) -> None:
    """The best node of every straddling row lies above its n*."""
    for c in CHUNKS:
        r, nstar = straddle(fleet.topo.n, c)
        row = rows_of(r // Q)[r % Q]
        assert int(np.argmax(row)) >= nstar, (c, int(np.argmax(row)), nstar)


def steps_pre(fleet: StepFleet) -> None:
    """The hub-anchored steps hold r* of both configurations; their patched set is far past shared memory (each
    anchor costs its closed neighbourhood); the straddle steps carry a consumed record just above each n*."""
    n = fleet.topo.n
    ts = np.asarray(fleet.blob[8:8 + 16 * len(fleet.steps)]).reshape(-1, 16)
    assert [int(x) for x in ts[:, 12]] == [Q * s for s in range(len(fleet.steps))]    # replica rows in step order
    for c in CHUNKS:
        r, nstar = straddle(n, c)
        assert r // Q in fleet.hub_steps, (c, r)
    for s in fleet.hub_steps:
        assert sg.patch_capacity(fleet.topo, fleet.steps[s]) > 16_384, s
        assert sg.exact_ok(fleet.steps[s], sg.amax_limit(fleet.topo)), s
    for s in STRADDLE:
        cons = [m for m, _ in fleet.steps[s].consumed]
        for pv in fleet.pivots:
            assert any(pv <= m < pv + 4 for m in cons), (s, pv)


def rerun_pre(fleet: Fleet, status_of) -> None:
    """Every group has two waves, 8 role rows then 1, and its oracle status is 1 (a replica of the first wave stays
    unplaced, so the plan hands it to the host-driven loop).  The loop keeps the first wave's 8 x G rows, so in both
    configurations the second wave's kept rows start past 2^31 floats and the first wave's straddle it.
    status_of(g) -> the oracle status of group g."""
    from gpu_util import plan_rows
    rows = plan_rows(fleet.blob, fleet.topo)
    ng = len(fleet.groups)
    assert sorted(rows) == sorted([(g, w) for g in range(ng) for w in (0, 1)])
    assert all(rows[(g, 1)] - rows[(g, 0)] == Q for g in range(ng))
    for g in fleet.distinct:
        assert status_of(g) == 1, g
    for c in CHUNKS:
        r, _ = straddle(fleet.topo.n, c)
        assert r < Q * ng and Q * ng * slab_stride(fleet.topo.n, c) > TWO31, c


# ---- oracles: one run per distinct group stands for the fleet

@dataclass
class Expect:
    assign: np.ndarray
    status: np.ndarray
    domain: np.ndarray
    score: np.ndarray = None
    alt_node: np.ndarray = None
    alt_score: np.ndarray = None


def expand(fleet, per: Dict[int, tuple], spans) -> Expect:
    """The whole fleet's outputs from per[rep] = (assign, status, domain, score, alt_node, alt_score) of each distinct
    group alone; spans[g] = group g's slice of the per-replica (or per-pod) outputs."""
    ng = len(fleet.rep)
    total = spans[-1].stop
    n_alt = next(iter(per.values()))[4].shape[1]
    e = Expect(np.empty(total, np.int32), np.empty(ng, np.int32), np.empty(ng, np.int32), np.empty(total, np.float32),
               np.empty((total, n_alt), np.int32), np.empty((total, n_alt), np.float32))
    for g in range(ng):
        a, s, d, sc, an, asc = per[fleet.rep[g]]
        e.assign[spans[g]], e.status[g], e.domain[g] = a, np.ravel(s)[0], np.ravel(d)[0]
        e.score[spans[g]], e.alt_node[spans[g]], e.alt_score[spans[g]] = sc, an, asc
    return e


def replica_spans(fleet) -> List[slice]:
    """Group g's slice of the per-replica outputs (GROUPS-blob order)."""
    out, off = [], 0
    for grp in fleet.groups:
        k = sum(r[1] for r in grp.roles)
        out.append(slice(off, off + k))
        off += k
    return out


def groups_oracle(fleet: Fleet, n_alt: int = 8, subset=None):
    """The wave loop and the ranked oracle on `subset` (default: the distinct groups), each group alone.  Returns
    (per[g] = six ranked outputs of group g, rows[(g, w)] = [roles][N] float32, topk[(g, w)] = [roles][32])."""
    import alternates_oracle
    from oracle import wave_loop
    og = wave_loop.groups_from_blob(fleet.blob)
    subset = fleet.distinct if subset is None else subset
    per, rows, topk = {}, {}, {}
    for g in subset:
        seen = []
        wave_loop.run_fleet(fleet.topo, [og[g]], want_matrix=True, want_topk=True,
                            on_wave=lambda w, act, blob, r: seen.append((w, r)))
        for w, r in seen:
            rows[(g, w)] = np.array(r["matrix"], copy=True)
            topk[(g, w)] = np.array(r["topk"], copy=True)
        per[g] = alternates_oracle.run_fleet_ranked(fleet.topo, [og[g]], n_alt)
    return per, rows, topk


def lw_spans(fleet: Fleet, rp) -> List[slice]:
    from lw_alternates_oracle import groups_of
    return [slice(X.pod0, X.pod0 + X.n_pods) for X in groups_of(fleet.blob, rp)]


def lw_oracle(fleet: Fleet, rp, n_alt: int = 8, subset=None):
    """run_lw_ranked on the owner-less snapshot with the co-location levels of lw_levels, group by group:
    per[g] = (assign, status, domain, score, alt_node, alt_score) of group g's pods."""
    import lw_oracle as lw
    from lw_alternates_oracle import run_lw_ranked
    topo, lvl = lw_topology(fleet.topo), lw_levels(fleet.topo)
    spans = lw_spans(fleet, rp)
    per = {}
    with lw.fast_domains():
        r = run_lw_ranked(topo, fleet.blob, rp, n_alt, level_domain=lvl,
                          groups=fleet.distinct if subset is None else subset)
    for g in (fleet.distinct if subset is None else subset):
        sl = spans[g]
        per[g] = (r[0][sl], int(r[1][g]), int(r[2][g]), r[3][sl], r[4][sl], r[5][sl])
    return per


def steps_oracle(fleet: StepFleet, subset=None):
    """The C oracle on each distinct step alone: per[s] = dict(assign, status, domain, matrix [8][N], topk [8][32])."""
    from oracle import placer as oracle_placer
    per = {}
    for s in (fleet.distinct if subset is None else subset):
        r = oracle_placer.place(fleet.topo, step_blob(fleet, s), want_matrix=True, want_topk=True)
        assert r["rc"] == 0, (s, r["rc"])
        per[s] = r
    return per


def need_bytes(rows: int, n: int, chunk_nodes: int = 0, copies: int = 1) -> int:
    """Device memory a case asks for: `copies` buffers of `rows` dense rows (DevBuf::reserve takes 1.25x), plus 2 GiB
    for the snapshot, the plan and the ranking's scratch."""
    return int(copies * rows * slab_stride(n, chunk_nodes) * 4 * 1.25) + (2 << 30)
