"""Designed cases of the all-gather selection limit tests (tests/test_gpu_allgather_limits.py on the device,
tests/test_allgather_limits_cases.py on the oracles alone; test infrastructure).

The all-gather scheme on node-axis shards (DESIGN.md §7): rank g selects, per role row, the top K_p keys of its slab
[bounds[g], bounds[g + 1]) (k_shard_select), the ranks' lists are all-gathered (by the caller, or by the library itself in
rbgtopo_run_staged_p2p), and every rank merges the world lists of K_p keys each (k_merge / merge_parts), with
K_p = min(replicas of roles 0..p, N).  An exclusive step without a fixed domain takes D* from the merged top-1 of its first
participating role, then a second exchange of lists restricted to D*, merged again in k_greedy.

Every builder returns (topo, blob, info) with info["worlds"] the worlds the case names.  Scores come from a bare snapshot
(alternates_limits_cases.bare_topo: no edge between nodes with room), so a node's score is set by its free capacity and by
the anchors on it.  The `*_pre` functions assert from the oracle's outputs and the slab bounds alone that the case still
reaches the edge it was designed for."""
from __future__ import annotations

import numpy as np

import alternates_limits_cases as al
from oracle import placer as oracle_placer
from oracle import wave_loop
from oracle.placer_ref import _key
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, STEP_GANG, BlobBuilder, Group, GroupsBuilder, Step
from shard_limits_cases import rank_of
from test_oracle_shard_alternates import slab_bounds
from test_shard_gloo import local_lists, merge_and_greedy

KS = 32
WORLDS = (3, 5, 8, 16)


def key_node(k):
    return 0xFFFFFFFF - (int(k) & 0xFFFFFFFF)


def topk_nodes(ref, rr):
    return [key_node(k) for k in ref["topk"][rr] if k]


def snapshot(n, free, domain=None):
    """A bare snapshot of n nodes: free[m] as given, and nodes n - 2, n - 1 set to 0 (bare_topo's one edge)."""
    f = np.asarray(free, np.int32).copy()
    assert len(f) == n
    f[n - 2:] = 0
    return al.bare_topo(f, domain)


def one_step(roles, **kw):
    P = len(roles)
    return BlobBuilder().add(Step(gid=kw.pop("gid", 1), roles=list(roles), pair=kw.pop("pair", np.eye(P, dtype=int).tolist()),
                                  **kw)).build()


# ---- 1. merge edges (merge_parts in k_merge, and in k_greedy for the restricted lists)

def _slab_nodes(bounds, r, k, gap=3):
    lo, hi = bounds[r], bounds[r + 1]
    nodes = [lo + 1 + gap * i for i in range(k)]
    assert nodes[-1] < hi - 2, (r, lo, hi)
    return nodes


def merge_case(name):
    kind, world = name.rsplit("_w", 1)
    world = int(world)
    n = 4096
    if kind == "empty300":
        n = 300
    elif kind == "ragged2049":
        n = 2049
    elif kind == "tiny":
        n = 20
    bounds = slab_bounds(n, world)
    free = np.full(n, 2, np.int32)
    roles = [(32, 1, 1, 0)]
    info = dict(worlds=(world,), kind=kind)
    if kind == "one_rank":                      # every winner of the role row in one rank's slab
        r = world // 2
        for m in _slab_nodes(bounds, r, 32):
            free[m] = 8
        info["rank"] = r
    elif kind == "two_per_rank":                # two winners in each of 16 ranks
        for r in range(world):
            for m in _slab_nodes(bounds, r, 2, gap=40):
                free[m] = 8
    elif kind == "ties":                        # 32 equal scores around a slab bound: node order decides the ranks
        b = bounds[world - 1]
        free[b - 16:b + 16] = 8
        info["bound"] = b
    elif kind == "ksmall":                      # K = 3 and 7: parts * K is no multiple of 32, winners in the last ranks
        roles = [(3, 1, 1, 0), (4, 1, 1, 0)]
        for i, m in enumerate(_slab_nodes(bounds, world - 1, 8, gap=5)):
            free[m] = 8 - (i % 2)
        for m in _slab_nodes(bounds, world - 2, 4, gap=7):
            free[m] = 7
    elif kind == "tiny":                        # N = 20 < 32 and K = N: only the last slab holds nodes
        roles = [(25, 1, 1, 0)]
        free[:] = np.arange(20) % 5 + 1
    elif kind == "short":                       # fewer feasible nodes in the cluster than K: the merge ends on a zero key
        roles = [(32, 3, 1, 0)]
        for r in range(world):
            for m in _slab_nodes(bounds, r, 20 // world + (r < 20 % world), gap=11):
                free[m] = 4
    elif kind in ("empty300", "ragged2049"):    # empty slabs first and in the middle / 128-node slabs, the last 129
        rng = np.random.default_rng(world + n)
        free[:] = rng.integers(1, 8, n)
        free[n - 19:n - 2:2] = 8                # winners in the last slab, up to its last node with room
        roles = [(25, 1, 1, 0), (7, 2, 3, 0)]
    else:
        raise KeyError(name)
    return snapshot(n, free), one_step(roles), info


MERGE_CASES = ([f"{k}_w{w}" for k in ("one_rank", "ties", "ksmall", "short") for w in WORLDS]
               + ["two_per_rank_w16", "tiny_w3", "tiny_w5", "empty300_w16", "ragged2049_w16"])


def merge_pre(name, topo, blob, info, ref=None):
    ref = oracle_placer.place(topo, blob) if ref is None else ref
    assert ref["rc"] == 0
    world = info["worlds"][0]
    bounds = slab_bounds(topo.n, world)
    kind = info["kind"]
    top = topk_nodes(ref, 0)
    ranks = [rank_of(bounds, m) for m in top]
    if kind == "one_rank":
        assert len(top) == 32 and set(ranks) == {info["rank"]}
    elif kind == "two_per_rank":
        assert len(top) == 32 and sorted(ranks) == sorted(list(range(16)) * 2)
    elif kind == "ties":
        S = ref["matrix"][0]
        assert len(top) == 32 and len({float(S[m]) for m in top}) == 1
        assert set(ranks) == {world - 2, world - 1} and top == list(range(info["bound"] - 16, info["bound"] + 16))
        assert float(S[info["bound"] + 16]) < float(S[top[0]])       # the next node loses on score, not on order
    elif kind == "ksmall":
        k = [len(topk_nodes(ref, rr)) for rr in range(2)]
        assert k == [3, 7] and all(world * kk % 32 for kk in k)
        assert set(rank_of(bounds, m) for m in topk_nodes(ref, 1)) >= {world - 1}
        assert all(rank_of(bounds, m) > 0 for m in topk_nodes(ref, 1))
    elif kind == "tiny":
        assert topo.n < 32 and len(top) == topo.n - 2 and all(lo == 0 for lo in bounds[:-1])   # K = N; 2 nodes have no room
    elif kind == "short":
        assert len(top) == 20 < 32 and (ref["assign"] < 0).sum() == 12 and ref["status"][0] == 1
    elif kind == "empty300":
        assert [hi - lo for lo, hi in zip(bounds, bounds[1:])][:6] == [0] * 6 and bounds[7] == bounds[8]
        assert rank_of(bounds, topk_nodes(ref, 0)[0]) == 15
    elif kind == "ragged2049":
        assert [hi - lo for lo, hi in zip(bounds, bounds[1:])] == [128] * 15 + [129]
        assert topo.n - 3 in topk_nodes(ref, 0) and rank_of(bounds, topo.n - 3) == 15
    return ref


# ---- 2. exclusive steps without a fixed domain

EXCL = STEP_EXCLUSIVE


def excl_case(name):
    kind, world = name.rsplit("_w", 1)
    world = int(world)
    n = 2049
    bounds = slab_bounds(n, world)
    rng = np.random.default_rng(len(kind) + world)
    free = rng.integers(1, 5, n).astype(np.int32)
    if kind == "split":       # domains of 128 nodes offset by 64: D* spans two slabs
        domain = ((np.arange(n) + 64) // 128).astype(np.int32)
    else:                     # domains of 64 nodes: every domain inside one slab
        domain = (np.arange(n) // 64).astype(np.int32)
    info = dict(worlds=(world,), kind=kind)
    anchors = []
    r_star = world - 1 if kind != "split" else world // 2
    x = bounds[r_star] + 5 if kind != "split" else bounds[r_star] - 3   # role 0's best node
    info["x"] = x
    pair = np.eye(3, dtype=int).tolist()
    if kind in ("far", "split", "opted_out"):
        # role 0 (exclusive) is drawn to x by its own anchor; role 2 (exclusive) prefers free-8 nodes in rank 0's slab;
        # role 1 is opted out (kind opted_out) or exclusive
        anchors = [(x, 0, 40)]
        free[x] = 4
        for m in range(bounds[0] + 2, bounds[0] + 12):
            free[m] = 8
        r1 = 0 if kind == "opted_out" else ROLE_EXCLUSIVE
        roles = [(3, 1, 2, ROLE_EXCLUSIVE), (4, 1, 2, r1), (5, 1, 2, ROLE_EXCLUSIVE)]
    elif kind == "later":      # the first role is opted out: the second decides D*
        for m in range(bounds[0] + 2, bounds[0] + 12):
            free[m] = 8
        anchors = [(x, 1, 40)]
        roles = [(4, 1, 2, 0), (6, 1, 2, ROLE_EXCLUSIVE)]
        pair = np.eye(2, dtype=int).tolist()
    elif kind == "none":       # nothing feasible anywhere: D* = -1
        roles = [(4, 9, 2, ROLE_EXCLUSIVE), (2, 9, 2, ROLE_EXCLUSIVE)]
        pair = np.eye(2, dtype=int).tolist()
    else:
        raise KeyError(name)
    topo = snapshot(n, free, domain)
    topo.domain_owner[:] = -1
    blob = one_step(roles, pair=pair, anchors=anchors, flags=EXCL)
    return topo, blob, info


EXCL_CASES = [f"{k}_w{w}" for k in ("far", "split", "opted_out", "later", "none") for w in WORLDS]


def excl_pre(name, topo, blob, info, ref=None):
    ref = oracle_placer.place(topo, blob) if ref is None else ref
    assert ref["rc"] == 0
    world = info["worlds"][0]
    bounds = slab_bounds(topo.n, world)
    kind = info["kind"]
    d = int(ref["domain"][0])
    if kind == "none":
        assert d == -1 and (ref["assign"] < 0).all() and ref["topk"].sum() == 0
        return ref
    x = info["x"]
    assert d == topo.domain[x] >= 0
    dom_nodes = np.nonzero(topo.domain == d)[0]
    dom_ranks = {rank_of(bounds, m) for m in dom_nodes}
    if kind == "split":
        assert len(dom_ranks) == 2
    else:
        assert len(dom_ranks) == 1 and rank_of(bounds, x) != 0     # every other rank's restricted list is empty
    excl_rows = {"far": slice(0, 12), "split": slice(0, 12), "opted_out": np.r_[0:3, 7:12], "later": slice(4, 10)}[kind]
    placed = ref["assign"][excl_rows]
    assert (placed >= 0).all() and (topo.domain[placed] == d).all()   # every exclusive replica inside D*
    if kind in ("far", "split", "opted_out"):
        # role 0 decides D* (its best node is x); the last exclusive role's unrestricted best lies outside D*, in rank
        # 0's slab, so its restricted list differs from the unrestricted one
        assert topk_nodes(ref, 0)[0] == x
        S2 = ref["matrix"][7]                                          # first replica row of role 2
        best2 = int(np.lexsort((np.arange(topo.n), -S2.astype(np.float64)))[0])
        assert topo.domain[best2] != d and rank_of(bounds, best2) == 0
        assert all(topo.domain[m] == d for m in topk_nodes(ref, 2))
        if kind == "opted_out":
            assert any(topo.domain[m] != d for m in ref["assign"][3:7])   # the opted-out role leaves D*
    if kind == "later":
        assert topk_nodes(ref, 1)[0] == x and rank_of(bounds, x) == world - 1
        assert any(topo.domain[m] != d for m in topk_nodes(ref, 0))
    return ref


# ---- 3. multi-wave plans

def _group(gid, roles, flags=0, anchors=(), pair=None):
    q = len(roles)
    return Group(gid=gid, roles=list(roles), pair=pair if pair is not None else np.ones((q, q), int).tolist(),
                 anchors=list(anchors), flags=flags)


def plan_case(name):
    n = 2049
    rng = np.random.default_rng(7 if name == "chain" else 8)
    free = rng.integers(1, 5, n).astype(np.int32)
    domain = (np.arange(n) // 100).astype(np.int32)
    gb = GroupsBuilder()
    if name == "chain":
        # an exclusive gang group of three levels (D* of wave 0 fixed into waves 1 and 2, its placements as anchors),
        # a plain group of two levels with 100 replicas at level 1 (four waves, past the exclusive group), a one-wave group
        gb.add(_group(1, [(0, 6, 1, ROLE_EXCLUSIVE), (1, 40, 1, ROLE_EXCLUSIVE), (2, 5, 1, 0)], EXCL | STEP_GANG))
        gb.add(_group(2, [(0, 9, 1, 0), (1, 100, 1, 0)]))
        gb.add(_group(3, [(0, 3, 2, 0)], anchors=[(1500, 0, 2)]))
    elif name == "gang_fail":
        # a gang group that fails in wave 0 (demand 9 > every free): its later steps are SKIP and push zero lists
        gb.add(_group(1, [(0, 4, 9, 0), (1, 12, 1, 0), (2, 33, 1, 0)], STEP_GANG))
        gb.add(_group(2, [(0, 5, 1, ROLE_EXCLUSIVE), (1, 7, 1, ROLE_EXCLUSIVE)], EXCL))
        gb.add(_group(3, [(0, 2, 1, 0), (1, 3, 1, 0), (2, 34, 1, 0)]))
    else:
        raise KeyError(name)
    topo = snapshot(n, free, domain)
    topo.domain_owner[:] = -1
    return topo, gb.build(), dict(worlds=(3, 5, 8), kind=name)


PLAN_CASES = ["chain", "gang_fail"]


def oracle_plan(topo, gblob):
    """The oracle's wave loop on a GROUPS blob: (states, per wave (wave, group indices, blob, oracle result))."""
    groups = wave_loop.groups_from_blob(gblob)
    index = {id(g): i for i, g in enumerate(groups)}
    waves = []
    states, _ = wave_loop.run_fleet(topo, groups, want_matrix=True, want_topk=True,
                                    on_wave=lambda w, act, blob, r: waves.append((w, [index[id(s.g)] for s in act], blob, r)))
    return states, waves


def plan_pre(name, topo, gblob, info, plan=None):
    states, waves = oracle_plan(topo, gblob) if plan is None else plan
    assert len(waves) >= 3
    if name == "chain":
        st = states[0]
        assert st.result()["status"] == 0 and st.result()["domain"] >= 0
        # waves 1 and 2 of the exclusive group ran with the fixed domain wave 0 chose, and with its placements as anchors
        for w, gis, blob, r in waves[1:3]:
            s = list(gis).index(0)
            assert int(blob[8 + 16 * s + 2]) == st.result()["domain"] and int(blob[8 + 16 * s + 7]) > 0
        assert sum(1 for w, gis, _, _ in waves if 1 in gis) >= 3    # the 40-replica level takes two waves
    else:
        assert states[0].result()["status"] == 2 and states[0].failed
        assert all(0 not in gis for w, gis, _, _ in waves[1:])        # later steps of the failed group are skipped
        assert len(states[0].waves) == 4
    return states, waves


# ---- the numpy shard protocol (tests/test_shard_gloo.py) at a world

def protocol(topo, blob, world, ref):
    """local lists per slab, merge, restricted reselect, merge + greedy: (assign, status, D*, merged lists)."""
    bounds = slab_bounds(topo.n, world)
    parts = [local_lists(ref["matrix"], topo, blob, lo, hi) for lo, hi in zip(bounds, bounds[1:])]
    merged, dstar = merge_and_greedy(topo, blob, parts, None)
    parts2 = [local_lists(ref["matrix"], topo, blob, lo, hi, dstar=dstar) for lo, hi in zip(bounds, bounds[1:])]
    assign, status, dstar = merge_and_greedy(topo, blob, parts, parts2)
    return assign, status, dstar, merged, parts, parts2


def protocol_topk(topo, blob, world, ref):
    """The final list of every role row the protocol leaves (restricted ones for exclusive roles of unknown D*)."""
    assign, status, dstar, merged, parts, parts2 = protocol(topo, blob, world, ref)
    ns = int(blob[2])
    out = np.zeros_like(ref["topk"])
    for s in range(ns):
        st = blob[8 + 16 * s: 8 + 16 * (s + 1)]
        flags, fixed, P, role_off, rr_off = int(st[1]), int(st[2]), int(st[3]), int(st[4]), int(st[13])
        roles = blob[role_off: role_off + 4 * P].reshape(P, 4)
        kacc = 0
        for p in range(P):
            kacc += int(roles[p, 0])
            keys = merged[(s, p)]
            if flags & STEP_EXCLUSIVE and fixed < 0 and roles[p, 3] & ROLE_EXCLUSIVE:
                keys = sorted((int(k) for part in parts2 for k in part[rr_off + p] if k), reverse=True)[:kacc]
            out[rr_off + p, :len(keys)] = keys
    return assign, status, dstar, out


def all_step_cases():
    return ([("merge", c) for c in MERGE_CASES] + [("excl", c) for c in EXCL_CASES])


def step_case(family, name):
    return merge_case(name) if family == "merge" else excl_case(name)


def step_pre(family, name, topo, blob, info, ref=None):
    return (merge_pre if family == "merge" else excl_pre)(name, topo, blob, info, ref)


# ---- peer bytes of one rbgtopo_run_staged_p2p pass

def phases_rows(blob_kind, blob, topo):
    """(phases, role rows) of every wave of a staged batch: one phase per wave, a second one for a wave with an exclusive
    step of unknown domain (a plan: with a step of an exclusive group)."""
    if blob_kind == "steps":
        ns = int(blob[2])
        excl = any(int(blob[8 + 16 * s + 1]) & STEP_EXCLUSIVE and int(blob[8 + 16 * s + 2]) < 0 for s in range(ns))
        return [(2 if excl else 1, max(1, int(blob[5])))]
    # every wave of every group is a step of the plan, those of a failed gang group included (they push zero lists)
    states = [wave_loop.GroupState(g) for g in wave_loop.groups_from_blob(blob)]
    out = []
    for w in range(max(len(s.waves) for s in states)):
        live = [s for s in states if w < len(s.waves)]
        excl = any(s.g.exclusive for s in live)
        out.append((2 if excl else 1, max(1, sum(len(s.waves[w]) for s in live))))
    return out


def peer_bytes(blob_kind, blob, topo, world):
    return sum(ph * rows * KS * 8 * (world - 1) for ph, rows in phases_rows(blob_kind, blob, topo))
