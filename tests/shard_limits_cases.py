"""Designed cases of the node-axis shard limit tests (tests/test_gpu_shard_limits.py on the device,
tests/test_oracle_shard_limits.py on the oracles alone; test infrastructure).  Every builder returns the snapshot, the
GROUPS blob and, for leader-worker cases, role_pods; the `*_pre` functions assert from the oracle's outputs and the
slab bounds alone that the case still hits the edge it was designed for.

Ranked alternates on shards (DESIGN.md §3.17): rank g ranks its slab [bounds[g], bounds[g + 1]) with
k_alternates_slab[_coloc], one thread per 4 slab-relative nodes (slab_thread_of), and writes the ALT_LIST best keys of
each job; k_alternates_merge reads the world · ALT_LIST gathered keys of a job with one warp, key i = position
i mod 9 of rank i div 9's list on lane i mod 32 (merge_lane_of).  Scores are set as in alternates_limits_cases: a bare
snapshot, S[m] = 8000 · (need · min(free[m], 8) + anchors on m) at every node with room.

Leader-worker placement on shards (§3.18): k_lw_assign_repl builds, per step, a patch table with one record per node
of the anchors' closed neighbourhoods and of the consumed records (npat), compacted from a bitmap of ceil(n / 32)
words in which thread t owns words [t · per, (t + 1) · per), per = ceil(words / 256)."""
from __future__ import annotations

import contextlib

import numpy as np

import alternates_limits_cases as al
import lw_oracle as lw
from oracle import placer as oracle_placer
from rbg_b200 import synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, Group
from test_oracle_lw_shards import HDR, SW, model_rows
from test_oracle_shard_alternates import ALT_LIST, best, shard_rank, slab_bounds

LW_THREADS = 256


def slab_thread_of(m, lo):
    """The k_alternates_slab thread that scans node m of the slab starting at lo."""
    return ((np.asarray(m) - lo) >> 2) & 255


def merge_lane_of(rank, pos):
    """The k_alternates_merge lane that reads position pos of rank's list."""
    return (ALT_LIST * rank + pos) % 32


def lane_keys(world, lane):
    """(rank, pos) of every gathered key lane `lane` reads at `world`."""
    return [(i // ALT_LIST, i % ALT_LIST) for i in range(lane, world * ALT_LIST, 32)]


def slab_lists(S, ok, bounds):
    return [best(S, lo + np.nonzero(ok[lo:hi])[0], ALT_LIST) for lo, hi in zip(bounds, bounds[1:])]


def winners(S, ok, bounds):
    """(rank, pos) in the gathered lists of each of the merged top ALT_LIST keys of a row, best first."""
    lists = slab_lists(S, ok, bounds)
    where = {int(m): (r, p) for r, lst in enumerate(lists) for p, m in enumerate(lst)}
    return [where[int(m)] for m in best(S, np.concatenate(lists), ALT_LIST)], lists


def rank_of(bounds, m):
    """The last w with bounds[w] <= m (the rank whose slab holds m)."""
    return max(w for w in range(len(bounds) - 1) if bounds[w] <= m)


def jobs(topo, gblob, exp, committed=False):
    """(row, candidate mask, own node) of every replica of a plain (or committed) ranked call of one-pod roles
    without exclusive groups, in assign order."""
    rows = al.oracle_rows(topo, gblob)
    out, i = [], 0
    for room, dem in al.room_after(topo, gblob, exp[0], committed=committed):
        for d in dem:
            out.append((rows[i], (rows[i] != -np.inf) & (room >= d), int(exp[0][i])))
            i += 1
    return out


def model_alternates(topo, gblob, exp, world, n_alt=8):
    """Alternates of every replica through the shard protocol (slab lists, rank-major merge) at `world`."""
    bounds = slab_bounds(topo.n, world)
    return [shard_rank(S, ok, own, n_alt, bounds) if own >= 0 else [] for S, ok, own in jobs(topo, gblob, exp)]


def one_job(anchors, n, free, roles=((0, 1, 1, 0),)):
    return al.bare_topo(free), al.build([Group(gid=1, roles=list(roles), pair=[[1] * len(roles)] * len(roles),
                                               anchors=anchors)])


# ---- 1. the merge lanes

LANE_CASES = {   # name: (world, n, the (rank, pos) of the nine winners, the replica's own (rank, pos))
    "lane0_w8": (8, 2048, [(0, 0)] + [(3, p) for p in range(6)] + [(7, 0), (7, 1)], (3, 0)),
    # at world 16 the five keys of lane 0 cannot all win: a key at list position p has p better keys of its own slab,
    # so (0,0) (3,5) (7,1) (10,6) (14,2) need 19 winners; the three of lowest position and their slab-mates win here
    "lane0_w16": (16, 4096, [(0, 0), (7, 0), (7, 1), (14, 0), (14, 1), (14, 2), (10, 0), (10, 1), (10, 2)], (10, 0)),
    "past32_w8": (8, 2048, [(4, 0), (4, 1), (5, 0), (5, 1), (6, 0), (6, 1), (7, 0), (7, 1), (7, 2)], (5, 0)),
    "one_rank_w8": (8, 2048, [(6, p) for p in range(9)], (6, 0)),
    "nine_ranks_w16": (16, 4096, [(r, 0) for r in range(7, 16)], (11, 0)),
}


def lanes_case(name):
    """One replica (demand 1, keeps room) on the own winner; winner (r, p) is node bounds[r] + 8 + 3p with anchor
    count 80 - 3p (the own one 99), so it is position p of rank r's list; twelve fillers per slab (counts 1..12) fill
    every list to ALT_LIST keys below the winners."""
    world, n, places, own = LANE_CASES[name]
    bounds = slab_bounds(n, world)
    free = np.zeros(n, np.int32)
    anchors = []
    for r, p in places:
        m = bounds[r] + 8 + 3 * p
        free[m] = 2
        anchors.append((m, 0, 99 if (r, p) == own else 80 - 3 * p))
    for lo in bounds[:-1]:
        for k in range(12):
            free[lo + 50 + 5 * k] = 2
            anchors.append((lo + 50 + 5 * k, 0, 1 + k))
    topo, gb = one_job(anchors, n, free)
    return topo, gb, dict(world=world, places=places, own=bounds[own[0]] + 8)


def lanes_pre(name, topo, gblob, info, exp=None):
    exp = al.ranked(topo, gblob) if exp is None else exp
    world, places = info["world"], info["places"]
    (S, ok, own), = jobs(topo, gblob, exp)
    assert own == info["own"]
    won, lists = winners(S, ok, slab_bounds(topo.n, world))
    assert sorted(won) == sorted(places), (won, places)
    assert all(len(lst) == ALT_LIST for lst in lists)                  # every list full: losers on every lane
    idx = [ALT_LIST * r + p for r, p in won]
    if name == "lane0_w8":
        assert set(lane_keys(8, 0)) <= set(won) and len(lane_keys(8, 0)) == 3
    elif name == "lane0_w16":
        assert len(lane_keys(16, 0)) == 5 and len(set(lane_keys(16, 0)) & set(won)) == 3
        assert {merge_lane_of(r, p) for r, p in [(0, 0), (7, 1), (14, 2)]} == {0}
    elif name == "past32_w8":
        assert min(idx) >= 32
    elif name == "one_rank_w8":
        assert len({r for r, _ in won}) == 1
    else:
        assert len({r for r, _ in won}) == 9 and min(idx) >= 32
    assert exp[4][0].tolist() == [int(m) for m in best(S, np.nonzero(ok)[0], 9) if m != own][:8]
    return exp


# ---- 2. empty slabs and the replica-score lookup

EMPTY_WORLDS = {3: 150, 4: 300, 5: 300, 8: 700}


def empty_targets(world):
    n = EMPTY_WORLDS[world]
    b = slab_bounds(n, world)
    return n, b, sorted({0, n - 1, n // 2} | {x for v in b[1:-1] if 0 < v < n for x in (v, v - 1)})


def empty_case(world):
    """One group (one replica, demand 1) per target node: the first and last node of every non-empty slab and n / 2.
    Its own node is its global best (count 99); its alternates are the next eight targets (counts 50..43), for even
    groups only those in other slabs; no other node has room."""
    n, b, targets = empty_targets(world)
    free = np.zeros(n, np.int32)
    free[targets] = 2
    groups = []
    for k, t in enumerate(targets):   # even groups: alternates only in other slabs
        others = [targets[(k + j) % len(targets)] for j in range(1, len(targets))]
        others = [m for m in others if k % 2 or rank_of(b, m) != rank_of(b, t)][:8]
        anchors = [(t, 0, 99)] + [(m, 0, 50 - j) for j, m in enumerate(others)]
        groups.append(Group(gid=10 + k, roles=[(0, 1, 1, 0)], pair=[[1]], anchors=anchors))
    return al.bare_topo(free), al.build(groups), dict(targets=targets)


def empty_pre(world, topo, gblob, info, exp=None):
    exp = al.ranked(topo, gblob) if exp is None else exp
    n, b, targets = empty_targets(world)
    assert b[0] == b[1]                                                        # an empty first slab
    assert any(b[w] == b[w + 1] for w in range(1, world))                      # and an empty middle one
    assert exp[0].tolist() == targets and (exp[3] > 0).all()
    nonempty = [w for w in range(world) if b[w] < b[w + 1]]
    assert all(b[w] in targets for w in nonempty)                               # first node of every slab
    assert all(b[w] - 1 in targets for w in nonempty if b[w] > 0)               # last node of the slab before
    assert any(b[w - 1] == b[w] for w in nonempty if w > 0)                     # a slab right after an empty one
    assert len(exp[0]) % 4 != 0 or world == 4                                   # ragged last merge CTA
    far = [r for r, own in enumerate(exp[0]) if exp[4][r][0] >= 0 and rank_of(b, exp[4][r][0]) != rank_of(b, own)]
    assert far or len(nonempty) == 1                            # the global best in another slab than the next best
    return exp


# ---- 3. the slab thread layouts at slab_lo mod 1024 != 0

LAYOUT_N = {2: 4500, 3: 7000}      # slab 1 starts at 2176 (world 2) and 2304 (world 3)


def layout_case(kind, own, world):
    lo = slab_bounds(LAYOUT_N[world], world)[1]
    return al.merge_case(kind, own, lo=lo, n_total=LAYOUT_N[world])


def layout_pre(kind, own, world, topo, gblob, info, exp=None):
    """The shifted case is the designed one node for node, and all its nodes lie in slab 1."""
    n = LAYOUT_N[world]
    b = slab_bounds(n, world)
    lo = b[1]
    assert lo % 1024 != 0 and b[2] - lo >= al.layout(kind)[0]
    base = al.merge_case(kind, own)
    e0 = al.merge_pre(kind, own, *base)
    exp = al.ranked(topo, gblob) if exp is None else exp
    assert np.array_equal(exp[0], e0[0] + lo)
    assert np.array_equal(exp[4], np.where(e0[4] >= 0, e0[4] + lo, -1))
    for k in (3, 5):
        assert np.array_equal(np.asarray(exp[k]).view(np.uint32), np.asarray(e0[k]).view(np.uint32))
    assert (slab_thread_of(info["win"], lo) == al.thread_of(np.asarray(info["win"]) - lo)).all()
    assert all(lo <= m < b[2] for m in info["win"] + [info["x"]])
    return exp


# ---- 4. ties and counts

def ties_case(world):
    """Twelve candidates of one score, six on each side of the middle slab bound."""
    n = 1100
    b = slab_bounds(n, world)[world // 2]
    free = np.zeros(n, np.int32)
    free[b - 6:b + 6] = 2
    topo, gb = one_job([], n, free)
    return topo, gb, dict(b=b)


def ties_pre(world, topo, gblob, info, exp=None):
    exp = al.ranked(topo, gblob) if exp is None else exp
    b = info["b"]
    assert exp[0][0] == b - 6 and exp[4][0].tolist() == list(range(b - 5, b + 3))
    assert (exp[5][0] == exp[3][0]).all()
    (S, ok, own), = jobs(topo, gblob, exp)
    assert ok.sum() > ALT_LIST and len(set(S[ok].tolist())) == 1
    assert {rank_of(slab_bounds(topo.n, world), m) for m in np.nonzero(ok)[0]} == {world // 2 - 1, world // 2}
    return exp


def zero_row_pre(world, topo, gblob, exp=None):
    """al.zero_row_case: a row of +0.0 over four non-empty slabs."""
    b = slab_bounds(topo.n, world)
    assert world == 4 and all(b[w] < b[w + 1] for w in range(world))
    return al.zero_row_pre(topo, gblob, exp)


COUNT_N, COUNT_WORLD = 1100, 4


def count_case(F):
    """The own node (count 99) in slab 1 and max(F - 1, 0) more candidates alternating between slabs 1 and 3; slabs 0
    and 2 hold no candidate.  Ranked at n_alt = F: fewer candidates than n_alt (F > 0)."""
    b = slab_bounds(COUNT_N, COUNT_WORLD)
    free = np.zeros(COUNT_N, np.int32)
    own = b[1] + 40
    nodes = [(b[1] if k % 2 == 0 else b[3]) + 60 + 4 * k for k in range(max(F - 1, 0))]
    free[[own] + nodes] = 2
    anchors = [(own, 0, 99)] + [(m, 0, 20 + k) for k, m in enumerate(nodes)]
    topo, gb = one_job(anchors, COUNT_N, free)
    return topo, gb, dict(own=own, nodes=nodes)


def count_pre(F, topo, gblob, info, exp=None):
    exp = al.ranked(topo, gblob) if exp is None else exp
    assert exp[0][0] == info["own"]
    k = int((exp[4][0] >= 0).sum())
    assert k == max(F - 1, 0) and (F == 0 or k < F)
    (S, ok, own), = jobs(topo, gblob, exp)
    lists = slab_lists(S, ok, slab_bounds(topo.n, COUNT_WORLD))
    assert len(lists[0]) == 0 and len(lists[2]) == 0
    return exp


def odd_case():
    """Three replicas (an odd compact replica count) on 2 048 nodes at world 8; all candidates lie in slabs 4..7."""
    n = 2048
    free = np.zeros(n, np.int32)
    nodes = np.arange(1030, n, 13)
    free[nodes] = 2
    anchors = [(int(m), 0, 1 + k % 40) for k, m in enumerate(nodes)]
    topo, gb = one_job(anchors, n, free, roles=((0, 3, 1, 0),))
    return topo, gb, {}


def odd_pre(topo, gblob, info, exp=None):
    exp = al.ranked(topo, gblob) if exp is None else exp
    assert len(exp[0]) % 2 == 1 and (exp[0] >= 0).all()
    b = slab_bounds(topo.n, 8)
    assert all(rank_of(b, m) >= 4 for m in exp[4].ravel() if m >= 0) and (exp[4] >= 0).all()
    return exp


def pods32_case():
    """One leader-worker replica of 32 pods (C = -1, demand 1) on 2 048 nodes: the 32 best of 60 one-pod nodes in
    slabs 4..7 take the pods; the others are every pod's alternates."""
    n = 2048
    free = np.zeros(n, np.int32)
    nodes = np.arange(1030, n, 16)[:60]
    free[nodes] = 1
    anchors = [(int(m), 0, 1 + k) for k, m in enumerate(nodes)]
    topo, gb = one_job(anchors, n, free)
    return topo, gb, np.array([(32, -1)], np.int32)


def lw_ranked_oracle(topo, gblob, rp, n_alt=8):
    from test_gpu_lw_limits import oracle_lw
    return oracle_lw(topo, gblob, np.asarray(rp, np.int32).reshape(-1, 2), None, n_alt)


def pods32_pre(topo, gblob, rp, exp=None):
    exp = lw_ranked_oracle(topo, gblob, rp) if exp is None else exp
    assert len(exp[0]) == 32 and (exp[0] >= 0).all() and len(set(exp[0].tolist())) == 32
    b = slab_bounds(topo.n, 8)
    assert (exp[4] >= 0).all() and all(rank_of(b, m) >= 4 for m in exp[4].ravel())
    return exp


# ---- 5. the slab room bitmap

BITMAP_N, BITMAP_WORLD = 3000, 3       # slab 1 = [896, 1920)


def slab_edges():
    b = slab_bounds(BITMAP_N, BITMAP_WORLD)
    lo, hi = b[1], b[2]
    return lo, hi, [lo, lo + 31, lo + 32, hi - 1], [lo - 1, hi]


def bitmap_case(pattern):
    """Role A (demand 3) puts one pod on each of slab 1's local bits 0, 31, 32 and len - 1 and on the nodes just
    outside it, leaving room 2 or 1 by `pattern`; role B (demand 2) takes node X and ranks the edge nodes next, but
    only those with room 2 fit it."""
    lo, hi, inside, outside = slab_edges()
    E = inside + outside
    x = (lo + hi) // 2
    free = np.zeros(BITMAP_N, np.int32)
    for k, m in enumerate(E):
        free[m] = 5 if (k + pattern) % 2 == 0 else 4
    free[x] = 8
    bg = np.arange(lo + 100, hi - 100, 97)[:10]
    free[bg] = 2
    anchors = [(m, 0, 25 + k) for k, m in enumerate(E)] + [(x, 1, 100)]
    g = Group(gid=7, roles=[(0, len(E), 3, 0), (0, 1, 2, 0)], pair=[[1, 0], [1, 1]], anchors=anchors)
    return al.bare_topo(free), al.build([g]), dict(E=E, x=x)


def bitmap_pre(pattern, topo, gblob, info, exp=None):
    exp = al.ranked(topo, gblob) if exp is None else exp
    E, x = info["E"], info["x"]
    a, an = exp[0], exp[4]
    k = len(E)
    assert sorted(a[:k].tolist()) == sorted(E) and a[k] == x
    room = al.room_after(topo, gblob, a)[0][0]
    fits, short = [m for m in E if room[m] == 2], [m for m in E if room[m] == 1]
    alts = an[k][an[k] >= 0]
    assert fits and short and set(fits) <= set(alts.tolist()) and not set(short) & set(alts.tolist())
    S = al.oracle_rows(topo, gblob)[k]
    assert all(S[m] > S[alts[-1]] for m in short)       # without the room test they would be listed
    lo, hi, inside, _ = slab_edges()
    assert [m - lo for m in inside] == [0, 31, 32, hi - lo - 1] and (hi - lo) % 32 == 0
    return exp


MANY_N, MANY_WORLD = 2100, 8


def many_used_case():
    """B (1 replica, demand 1, level 0) ranks its row; A (300 replicas of demand 2, level 1) fills nodes 3 + 7k, which
    lie in every slab at world 8; B's best-scored nodes are A's last twenty, past the 256th entry of the group's
    placement list."""
    free = np.zeros(MANY_N, np.int32)
    used = 3 + 7 * np.arange(300)
    free[used] = 2
    other = np.setdiff1d(np.arange(5, MANY_N, 11), used)[:50]
    free[other] = 1
    x = int(other[-1])
    anchors = [(int(m), 0, 50 + k) for k, m in enumerate(used[280:])] + [(x, 0, 100)]
    g = Group(gid=8, roles=[(0, 1, 1, 0), (1, 300, 2, 0)], pair=[[1, 0], [0, 1]], anchors=anchors)
    return al.bare_topo(free), al.build([g]), dict(x=x, late=used[280:].tolist())


def many_used_pre(topo, gblob, info, exp=None):
    exp = al.ranked(topo, gblob) if exp is None else exp
    a, an = exp[0], exp[4]
    used = np.unique(a[1:][a[1:] >= 0])
    b = slab_bounds(topo.n, MANY_WORLD)
    assert len(used) == 300 and a[0] == info["x"]
    assert {rank_of(b, m) for m in used} == set(range(MANY_WORLD))
    assert all(np.searchsorted(used, m) >= 256 for m in info["late"])
    S = al.oracle_rows(topo, gblob)[0]
    alts = an[0][an[0] >= 0]
    assert len(alts) == 8 and not set(alts.tolist()) & set(used.tolist())
    assert all(S[m] > S[alts[0]] for m in info["late"])
    return exp


# ---- 6. the patch table of k_lw_assign_repl

@contextlib.contextmanager
def scored_steps():
    """Every step blob the oracles score inside the block: [(topo, blob)] (oracle/placer.py's place)."""
    seen = []
    inner = oracle_placer.place

    def place(topo, blob, *a, **kw):
        seen.append((topo, np.asarray(blob, np.int64)))
        return inner(topo, blob, *a, **kw)
    oracle_placer.place = place
    try:
        yield seen
    finally:
        oracle_placer.place = inner


def steps_of(blob):
    """Per step of a step blob: dict(P, anchors [(m, q, c)], consumed [(m, amount)])."""
    out = []
    for s in range(int(blob[2])):
        st = blob[HDR + SW * s:HDR + SW * (s + 1)]
        na, nc = int(st[7]), int(st[9])
        out.append(dict(P=int(st[3]), anchors=blob[st[8]:st[8] + 3 * na].reshape(na, 3).tolist(),
                        consumed=blob[st[10]:st[10] + 2 * nc].reshape(nc, 2).tolist()))
    return out


def patched(topo, step):
    """The nodes of a step's patch table: the anchors' closed neighbourhoods and the consumed records."""
    rp, col = np.asarray(topo.row_ptr), np.asarray(topo.col_idx)
    nodes = {m for m, _ in step["consumed"]}
    for m, _, _ in step["anchors"]:
        nodes |= {m} | set(col[rp[m]:rp[m + 1]].tolist())
    return sorted(nodes)


def degree(topo, m):
    return int(topo.row_ptr[m + 1] - topo.row_ptr[m])


def word_owner(n, m):
    """(words, per, the thread that compacts node m's bitmap word)."""
    words = (n + 31) >> 5
    per = -(-words // LW_THREADS)
    return words, per, (m >> 5) // per


def hub_topo(n, hubs, free, seed=0):
    """A snapshot whose only edges join each hub h to its `deg` neighbours (weight 1 + position in h's adjacency,
    so the last neighbours weigh most); hubs: {h: neighbours}."""
    adj = [dict() for _ in range(n)]
    for h, nb in hubs.items():
        for k, m in enumerate(sorted(nb)):
            adj[h][m] = adj[m][h] = 1 + k
    deg = np.array([len(a) for a in adj])
    row_ptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int32)
    col = np.array([m for a in adj for m in sorted(a)], np.int32)
    w = np.array([a[m] for a in adj for m in sorted(a)], np.int32)
    dom = (np.arange(n) // 10).astype(np.int32)
    return synth.Topology(row_ptr, col, w, np.asarray(free, np.int32), dom, np.full(int(dom.max()) + 1, -1, np.int32))


HUB_N = 700


def hub_case(deg):
    """One replica of 4 pods anchored once at a hub (free 0) of `deg` neighbours with room 1: the pods take the four
    heaviest neighbours, the last of the hub's adjacency."""
    rng = np.random.default_rng(deg)
    h = 350
    nb = rng.choice(np.setdiff1d(np.arange(HUB_N), [h]), deg, replace=False)
    free = np.zeros(HUB_N, np.int32)
    free[np.arange(0, HUB_N, 3)] = 1
    free[nb] = 1
    free[h] = 0
    topo = hub_topo(HUB_N, {h: nb}, free)
    gb = al.build([Group(gid=1, roles=[(0, 1, 1, 0)], pair=[[1]], anchors=[(h, 0, 1)])])
    return topo, gb, np.array([(4, -1)], np.int32), dict(h=h, deg=deg)


def hub_pre(deg, topo, gblob, rp, info, exp=None):
    with scored_steps() as seen:
        exp = lw_ranked_oracle(topo, gblob, rp) if exp is None else exp
    h = info["h"]
    assert degree(topo, h) == deg
    adj = topo.col_idx[topo.row_ptr[h]:topo.row_ptr[h + 1]].tolist()
    pos = [adj.index(m) for m in exp[0]]
    assert sorted(pos) == list(range(deg - 4, deg)) and max(pos) >= 32 and (deg < 300 or min(pos) >= 256)
    (t, blob), = seen
    st, = steps_of(blob)
    assert len(patched(topo, st)) == deg + 1
    return exp


def five_anchors_case():
    """Five roles of one group anchored at one hub (five records (h, q, c)), a second hub whose neighbourhood
    overlaps the first's by twenty nodes: every warp of the prologue adds into the same records."""
    n = 400
    rng = np.random.default_rng(5)
    h1, h2 = 100, 300
    pool = rng.permutation(np.setdiff1d(np.arange(n), [h1, h2]))
    n1, n2 = pool[:40], np.concatenate([pool[20:40], pool[40:60]])
    free = np.zeros(n, np.int32)
    free[np.arange(1, n, 5)] = 1
    free[pool[:60]] = 2
    topo = hub_topo(n, {h1: n1, h2: n2}, free)
    roles = [(0, 1, 1, 0)] * 5
    pair = [[1 + (i + 2 * j) % 4 for j in range(5)] for i in range(5)]
    anchors = [(h1, q, 1 + q) for q in range(5)] + [(h2, 2, 2)]
    gb = al.build([Group(gid=1, roles=roles, pair=pair, anchors=anchors)])
    return topo, gb, np.array([(2, -1)] * 5, np.int32), dict(h=h1, h2=h2)


def five_anchors_pre(topo, gblob, rp, info, exp=None):
    with scored_steps() as seen:
        exp = lw_ranked_oracle(topo, gblob, rp) if exp is None else exp
    st = steps_of(seen[0][1])[0]
    on = [q for m, q, _ in st["anchors"] if m == info["h"]]
    assert len(on) == 5 and st["P"] == 5
    n1 = set(topo.col_idx[topo.row_ptr[info["h"]]:topo.row_ptr[info["h"] + 1]].tolist())
    n2 = set(topo.col_idx[topo.row_ptr[info["h2"]]:topo.row_ptr[info["h2"] + 1]].tolist())
    assert len(n1 & n2) == 20 and len(patched(topo, st)) == len(n1 | n2 | {info["h"], info["h2"]})
    assert (exp[0] >= 0).all() and set(exp[0].tolist()) <= n1 | n2
    return exp


def consumed_anchor_case():
    """Role A (level 0, S = 2) takes two nodes with room 3 in wave 0; role B (level 1, S = 2, paired with A) is
    staged in wave 1 with anchors on A's nodes, which carry consumed records too: B's best nodes are A's."""
    n = 300
    free = np.zeros(n, np.int32)
    free[np.arange(2, n, 4)] = 1
    hot = [41, 207]
    free[hot] = 3
    topo = synth.make_topology(n, seed=3, tiers=2, max_free=1)
    topo.free = free
    topo.domain_owner[:] = -1
    gb = al.build([Group(gid=1, roles=[(0, 1, 1, 0), (1, 1, 1, 0)], pair=[[1, 0], [40, 1]])])
    rp = np.array([(2, -1), (2, -1)], np.int32)
    return topo, gb, rp, dict(hot=hot)


def consumed_anchor_pre(topo, gblob, rp, info, exp=None):
    with scored_steps() as seen:
        exp = lw_ranked_oracle(topo, gblob, rp) if exp is None else exp
    a = exp[0]
    assert set(a[:2].tolist()) <= set(info["hot"])
    assert set(a[2:].tolist()) & set(a[:2].tolist())                   # B on a node it is anchored at and that A used
    st = next(st for _, b in seen for st in steps_of(b) if st["consumed"])
    both = {m for m, _, _ in st["anchors"]} & {m for m, _ in st["consumed"]}
    assert both == set(a[:2].tolist())
    return exp


def committed_consumed_case():
    """A committed batch: group 1 (demand 8) fills node 55, the best node by base; group 2 (exclusive, demand 2, no
    anchor) sees node 55 as a consumed record without an anchor, so its domain D* comes from node 77 (domain 7),
    not from 55's domain 5, where other nodes still have room."""
    n = 200
    topo = synth.make_topology(n, seed=4, tiers=2, max_free=1)
    free = np.zeros(n, np.int32)
    free[np.arange(1, n, 6)] = 2
    free[[51, 52, 53]] = 2
    free[55], free[77] = 8, 7
    topo.free = free
    topo.domain = (np.arange(n) // 10).astype(np.int32)
    topo.domain_owner = np.full(20, -1, np.int32)
    gb = al.build([Group(gid=1, roles=[(0, 1, 8, 0)], pair=[[1]]),
                   Group(gid=2, roles=[(0, 1, 2, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE)])
    return topo, gb, np.array([(1, -1), (2, -1)], np.int32), {}


def committed_oracle(topo, gblob, rp):
    from lw_committed_oracle import run_lw_committed
    with lw.fast_domains():
        return run_lw_committed(topo, gblob, np.asarray(rp, np.int32).reshape(-1, 2))


def committed_consumed_pre(topo, gblob, rp, info, exp=None):
    from test_oracle_lw_shards import base_of
    exp = committed_oracle(topo, gblob, rp) if exp is None else exp
    a, s, d = exp
    base = np.where(topo.free >= 2, base_of(topo), -1)
    assert int(np.argmax(base)) == 55 and a[0] == 55 and d[1] == 7 and (a[1:] >= 0).all()
    assert (np.asarray(topo.domain)[a[1:]] == 7).all()
    return exp


def mixed_width_case():
    """One wave of two steps: an 8-role group (P = 8, records 2 + 8 wide) and a 1-role group (P = 1) whose records
    are read at the same width; both anchored at hubs."""
    n = 500
    rng = np.random.default_rng(8)
    hubs = {10: rng.choice(np.arange(20, 250), 40, replace=False),
            400: rng.choice(np.arange(250, 390), 40, replace=False)}
    free = np.zeros(n, np.int32)
    free[np.arange(2, n, 3)] = 2
    for nb in hubs.values():
        free[nb] = 2
    topo = hub_topo(n, hubs, free)
    g8 = Group(gid=1, roles=[(0, 1, 1, 0)] * 8, pair=[[1 + (i * j) % 3 for j in range(8)] for i in range(8)],
               anchors=[(10, q, 1) for q in range(0, 8, 3)])
    g1 = Group(gid=2, roles=[(0, 1, 1, 0)], pair=[[1]], anchors=[(400, 0, 2)])
    return topo, al.build([g8, g1]), np.array([(1, -1)] * 8 + [(3, -1)], np.int32), {}


def mixed_width_pre(topo, gblob, rp, info, exp=None):
    with scored_steps() as seen:
        exp = lw_ranked_oracle(topo, gblob, rp) if exp is None else exp
    sts = steps_of(seen[0][1])
    assert sorted(st["P"] for st in sts) == [1, 8] and all(len(patched(topo, st)) > 0 for st in sts)
    assert (exp[0][8:] >= 0).all() and set(exp[0][8:].tolist()) <= set(topo.col_idx[topo.row_ptr[400]:topo.row_ptr[401]].tolist())
    return exp


def empty_table_case():
    """One wave of three steps: the middle group has no anchors and, in its first wave, no consumed records (an
    empty table); its neighbours have tables."""
    topo, gb0, _, _ = hub_case(33)
    free = topo.free.copy()
    free[::2] = np.maximum(free[::2], 1)
    topo = synth.Topology(topo.row_ptr, topo.col_idx, topo.edge_w, free, topo.domain, topo.domain_owner)
    gb = al.build([Group(gid=1, roles=[(0, 1, 1, 0)], pair=[[1]], anchors=[(350, 0, 1)]),
                   Group(gid=2, roles=[(0, 1, 1, 0)], pair=[[1]]),
                   Group(gid=3, roles=[(0, 1, 1, 0)], pair=[[1]], anchors=[(350, 0, 2)])])
    return topo, gb, np.array([(4, -1), (3, -1), (2, -1)], np.int32), {}


def empty_table_pre(topo, gblob, rp, info, exp=None):
    with scored_steps() as seen:
        exp = lw_ranked_oracle(topo, gblob, rp) if exp is None else exp
    sts = steps_of(seen[0][1])
    assert len(sts) == 3 and [len(patched(topo, st)) for st in sts] == [34, 0, 34]
    assert (exp[0] >= 0).all()
    return exp


LAST_NS = [31, 33, 8192, 8193]


def last_word_case(n):
    """Anchors at node n - 1 (room 1): the patched node sits in the last bitmap word, which is ragged for 33 and 8193
    (8193: 257 words, two per thread for the first 129 threads); only its anchor delta makes it a pod's node."""
    topo = synth.make_topology(n, seed=n, tiers=1 if n < 64 else 2, max_free=1)
    topo.domain_owner[:] = -1
    topo.free[n - 1] = 1
    gb = al.build([Group(gid=1, roles=[(0, 1, 1, 0)], pair=[[1]], anchors=[(n - 1, 0, 3)])])
    return topo, gb, np.array([(2, -1)], np.int32), {}


def last_word_pre(n, topo, gblob, rp, info, exp=None):
    with scored_steps() as seen:
        exp = lw_ranked_oracle(topo, gblob, rp) if exp is None else exp
    words, per, t = word_owner(n, n - 1)
    assert (n - 1) >> 5 == words - 1
    assert (words, per, t) == {31: (1, 1, 0), 33: (2, 1, 1), 8192: (256, 1, 255), 8193: (257, 2, 128)}[n]
    st, = steps_of(seen[0][1])
    assert len(patched(topo, st)) == degree(topo, n - 1) + 1
    assert n - 1 in exp[0].tolist()
    from test_oracle_lw_shards import base_of
    base = np.where(topo.free >= 1, base_of(topo), -1)
    assert int(np.argmax(base)) != n - 1                 # without its delta, another node outranks n - 1
    return exp


# ---- the lists the suites run

LW_CASES = ["hub33", "hub300", "five_anchors", "consumed_anchor", "mixed_width", "empty_table"] + \
    [f"last_word_{n}" for n in LAST_NS] + ["pods32"]
LW_WORLDS = (2, 3, 8)


def lw_case(name):
    """(topo, blob, role_pods, pre) of a leader-worker designed case; pre(exp=None) returns the ranked oracle."""
    if name.startswith("hub"):
        deg = int(name[3:])
        t, g, rp, info = hub_case(deg)
        return t, g, rp, lambda exp=None: hub_pre(deg, t, g, rp, info, exp)
    if name.startswith("last_word_"):
        n = int(name.split("_")[-1])
        t, g, rp, info = last_word_case(n)
        return t, g, rp, lambda exp=None: last_word_pre(n, t, g, rp, info, exp)
    if name == "pods32":
        t, g, rp = pods32_case()
        return t, g, rp, lambda exp=None: pods32_pre(t, g, rp, exp)
    build, pre = {"five_anchors": (five_anchors_case, five_anchors_pre),
                  "consumed_anchor": (consumed_anchor_case, consumed_anchor_pre),
                  "mixed_width": (mixed_width_case, mixed_width_pre),
                  "empty_table": (empty_table_case, empty_table_pre)}[name]
    t, g, rp, info = build()
    return t, g, rp, lambda exp=None: pre(t, g, rp, info, exp)


def alt_cases():
    """[(name, worlds, n_alts, builder() -> (topo, blob, pre(exp=None)))] of the one-pod ranked designed cases."""
    out = []

    def add(name, worlds, mk, pre, n_alts=(0, 1, 3, 8)):
        def make():
            t, g, info = mk()
            return t, g, lambda exp=None: pre(t, g, info, exp)
        out.append((name, worlds, n_alts, make))
    for name, (world, *_rest) in LANE_CASES.items():
        add(name, (world,), lambda name=name: lanes_case(name), lambda t, g, i, e, name=name: lanes_pre(name, t, g, i, e))
    for W in EMPTY_WORLDS:
        add(f"empty_w{W}", (W,), lambda W=W: empty_case(W), lambda t, g, i, e, W=W: empty_pre(W, t, g, i, e))
    for W in LAYOUT_N:
        for kind in al.MERGE_KINDS:
            for own in al.OWN:
                add(f"layout_{kind}_{own}_w{W}", (W,), lambda k=kind, o=own, W=W: layout_case(k, o, W),
                    lambda t, g, i, e, k=kind, o=own, W=W: layout_pre(k, o, W, t, g, i, e))
    for W in (4, 8):
        add(f"ties_w{W}", (W,), lambda W=W: ties_case(W), lambda t, g, i, e, W=W: ties_pre(W, t, g, i, e))
    add("zero_row_w4", (4,), lambda: (*al.zero_row_case(), None), lambda t, g, i, e: zero_row_pre(4, t, g, e))
    for F in range(9):
        add(f"count_{F}", (COUNT_WORLD,), lambda F=F: count_case(F), lambda t, g, i, e, F=F: count_pre(F, t, g, i, e),
            n_alts=tuple(sorted({F, 0, 1, 3, 8})))
    add("odd_replicas_w8", (8,), odd_case, odd_pre)
    for p in (0, 1):
        add(f"bitmap_{p}", (BITMAP_WORLD,), lambda p=p: bitmap_case(p), lambda t, g, i, e, p=p: bitmap_pre(p, t, g, i, e))
    add("many_used_w8", (MANY_WORLD,), many_used_case, many_used_pre)
    return out


ALT_NAMES = [c[0] for c in alt_cases()]


def alt_case(name):
    return next(c for c in alt_cases() if c[0] == name)
