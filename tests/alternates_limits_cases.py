"""Designed cases of the ranked-alternates limit tests (tests/test_gpu_alternates_limits.py on the device,
tests/test_oracle_alternates_limits.py on the oracle alone; test infrastructure).  Every builder returns the snapshot
and GROUPS blob of one case; the `*_pre` functions assert, from the oracle's outputs only, that the case still hits
the edge it was designed for.

Scores are controlled with a bare snapshot: one edge of weight 1 between two nodes without room, so a role row is
S[m] = 8000 · (need · min(free[m], 8) + Σ_q pair[ρ][q] · anchors(m, q)) at every node with room, and anchors set any
order we want.  k_alternates reads a row with 16-byte loads: thread t of the 256 scans nodes 4t + 1024i + j, so the
thread of node m is (m >> 2) & 255, its warp that >> 5 and its lane that & 31."""
from __future__ import annotations

import numpy as np

import committed_alternates_oracle as cao
import committed_oracle as co
import levels_oracle as lo
from alternates_oracle import run_fleet_ranked
from oracle import wave_loop
from rbg_b200 import synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, STEP_GANG, Group, GroupsBuilder

ALT_LIST = 9                      # the per-thread top list: n_alt = 8 plus the replica's own node
BITMAP_NODES = 200 * 1024 * 8     # the room bitmap's ceiling (200 KB of shared memory, one bit per node)
REPLAY_FLOATS = 1 << 28           # a committed replay chunk holds at most 1 GiB of rows
KEYS = [f"example.com/level-{L}" for L in range(8)]


def build(groups):
    gb = GroupsBuilder()
    for g in groups:
        gb.add(g)
    return gb.build()


def bare_topo(free, domain=None):
    """A snapshot whose only edge (weight 1) joins the two lowest nodes with free 0."""
    free = np.asarray(free, np.int32)
    n = len(free)
    a, b = (int(x) for x in np.nonzero(free == 0)[0][:2])
    deg = np.zeros(n, np.int64)
    deg[[a, b]] = 1
    row_ptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int32)
    dom = np.zeros(n, np.int32) if domain is None else np.asarray(domain, np.int32)
    return synth.Topology(row_ptr, np.array([b, a], np.int32), np.array([1, 1], np.int32), free, dom,
                          np.full(int(dom.max()) + 1, -1, np.int32))


def thread_of(m):
    return (np.asarray(m) >> 2) & 255


def warp_of(m):
    return thread_of(m) >> 5


def lane_of(m):
    return thread_of(m) & 31


def oracle_rows(topo, gblob):
    """The dense row of every replica (GROUPS-blob order) in the snapshot wave loop of place_groups_ranked."""
    rows = {}

    def on_wave(w, active, blob, r):
        off = 0
        for s in active:
            for ri, ordinal, cnt in s.waves[w]:
                for c in range(cnt):
                    rows[(s.g.name, ri, ordinal + c)] = np.array(r["matrix"][off], np.float32)
                off += cnt

    states, _ = wave_loop.run_fleet(topo, wave_loop.groups_from_blob(gblob), want_matrix=True, on_wave=on_wave)
    return [rows[(s.g.name, ri, s.first[ri] + c)] for s in states for ri in s.order for c in range(s.pending[ri])]


def row_rank(S, m):
    """How many nodes of row S outrank node m by key(score, node)."""
    fin = np.nonzero(S != -np.inf)[0]
    return int(((S[fin] > S[m]) | ((S[fin] == S[m]) & (fin < m))).sum())


def ranked(topo, gblob, n_alt=8):
    return run_fleet_ranked(topo, wave_loop.groups_from_blob(gblob), n_alt)


def room_after(topo, gblob, a, committed=False):
    """free - (demand placed on each node) per group (snapshot) or over the whole batch (committed), per replica."""
    gb = np.asarray(gblob)
    free = np.asarray(topo.free, np.int64)
    out, used_b, per = [], np.zeros(len(free), np.int64), []
    for g in range(int(gb[2])):
        q, role_off, pod0 = int(gb[8 + 12 * g + 3]), int(gb[8 + 12 * g + 4]), int(gb[8 + 12 * g + 8])
        used = np.zeros(len(free), np.int64)
        i = pod0
        dem = []
        for r in range(q):
            for _ in range(int(gb[role_off + 4 * r + 1])):
                dem.append(int(gb[role_off + 4 * r + 2]))
                if a[i] >= 0:
                    used[a[i]] += dem[-1]
                i += 1
        used_b += used
        per.append((used, dem))
    for used, dem in per:
        out.append((free - (used_b if committed else used), dem))
    return out


# ---- 1. the top-list merge

MERGE_KINDS = ["thread0", "warp", "per_warp", "warp7"]
OWN = ["rank0", "rank8", "full"]


def layout(kind):
    """(N, the nine winner nodes) of a stride layout."""
    if kind == "thread0":   # thread 0's whole stride set at N = 2049: {0..3, 1024..1027, 2048}
        return 2049, [1024 * i + j for i in range(3) for j in range(4)][:9]
    if kind == "warp":      # warp 2, nine lanes, both passes of the row
        return 2050, [4 * (64 + l) + (l % 4) + 1024 * (l % 2) for l in (0, 3, 5, 8, 13, 17, 22, 26, 31)]
    if kind == "per_warp":  # one node in each warp, the ninth in warp 0's second pass (node 1026 of 1027)
        return 1027, [128 * w + 4 * ((5 * w) % 32) + (w % 4) for w in range(8)] + [1026]
    assert kind == "warp7"
    return 2051, [4 * (224 + l) + (l % 4) + 1024 * (l % 2) for l in (1, 2, 4, 7, 11, 16, 20, 29, 31)]


def layout_holds(kind, nodes):
    nodes = np.asarray(sorted(nodes))
    if kind == "thread0":
        return (thread_of(nodes) == 0).all()
    if kind == "warp":
        return len(set(warp_of(nodes).tolist())) == 1 and len(set(lane_of(nodes).tolist())) == len(nodes)
    if kind == "per_warp":   # every warp, or (eight of the nine) all but one, with one warp holding two
        return len(set(warp_of(nodes).tolist())) == min(8, len(nodes) - 1)
    return (warp_of(nodes) == 7).all()


def merge_case(kind, own, lo=0, n_total=None):
    """One group.  rank0: one replica (demand 1) on the best winner, which keeps room, so the nine winners are its
    node and eight alternates.  rank8: eight replicas of demand 2 fill eight better filler nodes first, then one of
    demand 1 (the designated job, row rank 8) takes the best winner and keeps room.  full: the replica's node
    outranks everything but has room for it alone.  Six lower tail candidates sit elsewhere in the row.
    lo / n_total: the same case shifted to nodes lo .. lo + N of a snapshot of n_total nodes (free 0 elsewhere)."""
    n, win = layout(kind)
    if lo or n_total is not None:
        topo, gb, info = merge_case(kind, own)
        free = np.zeros(n_total, np.int32)
        free[lo:lo + n] = topo.free
        gb = gb.copy()
        na, anchor_off = int(gb[8 + 6]), int(gb[8 + 7])       # the one group's anchors: (node, role, count)
        gb[anchor_off:anchor_off + 3 * na:3] += lo
        return bare_topo(free), gb, dict(win=[m + lo for m in info["win"]], fill=info["fill"] + lo, x=info["x"] + lo)
    rng = np.random.default_rng(MERGE_KINDS.index(kind) * 10 + OWN.index(own))
    rest = np.setdiff1d(np.arange(2, n - 1), win)
    pick = rng.choice(rest, 15, replace=False)
    fill, tail, x = pick[:8], pick[8:14], int(pick[14])
    free = np.zeros(n, np.int32)
    free[win] = 2
    free[tail] = 2
    anchors = [(int(m), 0, 30 + 3 * int(p)) for m, p in zip(win, rng.permutation(9))]
    anchors += [(int(m), 0, 1 + k) for k, m in enumerate(tail)]
    if own == "rank8":
        free[fill] = 2
        anchors += [(int(m), 0, 60 + k) for k, m in enumerate(fill)]
        g = Group(gid=1, roles=[(0, 8, 2, 0), (0, 1, 1, 0)], pair=[[1, 1], [1, 1]], anchors=anchors)
    else:
        if own == "full":
            free[x] = 1
            anchors.append((x, 0, 70))
        g = Group(gid=1, roles=[(0, 1, 1, 0)], pair=[[1]], anchors=anchors)
    return bare_topo(free), build([g]), dict(win=win, fill=fill, x=x)


def merge_pre(kind, own, topo, gblob, info, exp=None):
    exp = ranked(topo, gblob) if exp is None else exp
    a, s, _, _, an, _ = exp
    r = len(a) - 1                                  # the designated job's replica
    room = room_after(topo, gblob, a)[0][0]
    top = set(an[r][an[r] >= 0].tolist())
    assert len(top) == 8, (kind, own, an[r])
    if own == "full":
        assert top < set(info["win"]) and layout_holds(kind, info["win"])
        assert a[r] == info["x"] and room[a[r]] == 0 and top <= set(info["win"])
    else:
        assert room[a[r]] >= 1 and top | {int(a[r])} == set(info["win"]), (a, an[r])
        assert layout_holds(kind, top | {int(a[r])})
        if own == "rank8":
            S = oracle_rows(topo, gblob)[r]
            assert sorted(a[:8].tolist()) == sorted(info["fill"].tolist()) and row_rank(S, a[r]) == 8
    return exp


def stack_case(demand):
    """One job of 32 replicas: eleven nodes with room for three (demand 1) take them three by three, the last keeps
    room for one; ten lower nodes with room for one.  Demand 0: all 32 on the best node."""
    n = 1030
    rng = np.random.default_rng(40 + demand)
    nodes = rng.choice(np.arange(2, n), 21, replace=False)
    free = np.zeros(n, np.int32)
    free[nodes[:11]] = 3
    free[nodes[11:]] = 1
    anchors = [(int(m), 0, 40 + k) for k, m in enumerate(nodes[:11])] + [(int(m), 0, 10 + k) for k, m in
                                                                          enumerate(nodes[11:])]
    return bare_topo(free), build([Group(gid=3, roles=[(0, 32, demand, 0)], pair=[[1]], anchors=anchors)])


def stack_pre(demand, topo, gblob, exp=None):
    exp = ranked(topo, gblob) if exp is None else exp
    a, an = exp[0], exp[4]
    room = room_after(topo, gblob, a)[0][0]
    assert len(a) == 32 and (a >= 0).all()
    if demand == 0:
        assert len(set(a.tolist())) == 1
    else:
        keep = [m for m in set(a.tolist()) if room[m] >= 1]
        assert len(set(a.tolist())) == 11 and len(keep) == 1, a
        assert all(keep[0] in an[r] for r in range(32) if a[r] != keep[0])
    return exp


def ties_case():
    """Twelve nodes with room, scattered over the warps, all with the same score."""
    n = 1100
    nodes = [5, 130, 131, 260, 400, 515, 640, 777, 900, 1024, 1030, 1099]
    free = np.zeros(n, np.int32)
    free[nodes] = 2
    return bare_topo(free), build([Group(gid=4, roles=[(0, 1, 1, 0)], pair=[[1]])]), nodes


def ties_pre(topo, gblob, nodes, exp=None):
    exp = ranked(topo, gblob) if exp is None else exp
    a, sc, an, asc = exp[0], exp[3], exp[4], exp[5]
    assert a[0] == nodes[0] and an[0].tolist() == nodes[1:9] and (asc[0] == sc[0]).all()
    return exp


def zero_row_case():
    """A demand-0 role with need 0 (pair [[0]]) and no anchors: a row of +0.0 at every node."""
    n = 1001
    free = np.random.default_rng(5).integers(0, 4, n).astype(np.int32)
    free[:2] = 0
    return bare_topo(free), build([Group(gid=5, roles=[(0, 1, 0, 0)], pair=[[0]])])


def zero_row_pre(topo, gblob, exp=None):
    exp = ranked(topo, gblob) if exp is None else exp
    S = oracle_rows(topo, gblob)[0]
    assert (S.view(np.uint32) == 0).all()
    assert exp[0][0] == 0 and exp[4][0].tolist() == list(range(1, 9)) and (exp[5][0].view(np.uint32) == 0).all()
    return exp


def counts(F):
    return [F - 1, F, F + 1] if F > 0 else [0, 1]


def count_case(F):
    """Exclusive groups fixed to domains 0, 1, 2 (32 nodes each, N = 101): group k's replica takes its domain's best
    node and keeps room; the domain holds exactly counts(F)[k] more candidates (the other domains' nodes have room too
    but are outside the domain)."""
    n = 101
    dom = np.minimum(np.arange(n) // 32, 3)
    free = np.zeros(n, np.int32)
    groups = []
    for k, m in enumerate(counts(F)):
        nodes = 32 * k + 2 + np.arange(m + 1) * 3
        free[nodes] = 2
        anchors = [(int(nodes[0]), 0, 40)] + [(int(x), 0, 10 + (7 * j) % 11) for j, x in enumerate(nodes[1:])]
        groups.append(Group(gid=10 + k, roles=[(0, 1, 1, ROLE_EXCLUSIVE)], pair=[[1]], anchors=anchors,
                            flags=STEP_EXCLUSIVE, fixed_domain=k))
    return bare_topo(free, dom), build(groups)


def count_pre(F, topo, gblob, exp=None):
    exp = ranked(topo, gblob, 8) if exp is None else exp
    for k, m in enumerate(counts(F)):
        assert exp[0][k] == 32 * k + 2 and (exp[4][k] >= 0).sum() == min(m, 8), (k, exp[4][k])
    return exp


# ---- 2. the room bitmap

BITMAP_NS = [97, 130, 131, 1057]   # N = 1, 2, 3 (mod 4) and 1 (mod 32)


def edge_nodes(n):
    return [0, 31, 32, 63, n - 1]


def bitmap_case(n, pattern, level=0):
    """One wave of three roles.  A (5 replicas, demand 3) lands one replica on each edge node, leaving room 2 or 1 by
    `pattern`; B (demand 2) then takes node X and ranks the edge nodes next, but only those left with room 2 have
    room for it; D (demand 0, need 1) ranks every node.  level > 0: the group is exclusive at that level (A and B
    take part, D opts out)."""
    E = edge_nodes(n)
    x = n // 2 + 1
    free = np.zeros(n, np.int32)
    for k, m in enumerate(E):
        free[m] = 5 if (k + pattern) % 2 == 0 else 4
    free[x] = 8
    bg = [m for m in range(2, n - 1) if m not in E and m != x][5::max(1, n // 12)][:10]
    free[bg] = 2
    anchors = [(m, 0, 25 + k) for k, m in enumerate(E)] + [(x, 1, 100)]
    fl = ROLE_EXCLUSIVE if level else 0
    g = Group(gid=7, roles=[(0, 5, 3, fl), (0, 1, 2, fl), (0, 1, 0, 0)], pair=[[1, 0, 0], [1, 1, 0], [0, 0, 1]],
              anchors=anchors, flags=STEP_EXCLUSIVE if level else 0, level=level)
    return bare_topo(free), build([g]), dict(E=E, x=x)


def bitmap_pre(topo, gblob, info, exp=None):
    exp = ranked(topo, gblob) if exp is None else exp
    a, an = exp[0], exp[4]
    room = room_after(topo, gblob, a)[0][0]
    E = info["E"]
    assert sorted(a[:5].tolist()) == sorted(E) and a[5] == info["x"]
    fits = [m for m in E if room[m] == 2]
    short = [m for m in E if room[m] == 1]
    assert fits and short
    S = oracle_rows(topo, gblob)[5]
    alts = an[5][an[5] >= 0]
    assert set(fits) <= set(alts.tolist()) and not set(short) & set(alts.tolist())
    assert all(S[m] > S[alts[-1]] for m in short)     # without the room test they would be listed
    return exp


def many_used_case():
    """B (1 replica, demand 1, level 0) ranks its row before A (300 replicas of demand 2, level 1, ten waves) fills
    nodes 0..299: B's best-scored nodes 280..299 sit past the 256th entry of the group's placement list."""
    n = 700
    free = np.zeros(n, np.int32)
    free[:300] = 2
    free[300:350] = 1
    x = 650
    free[x] = 1
    anchors = [(m, 0, 50 + m - 280) for m in range(280, 300)] + [(x, 0, 100)]
    free[[698, 699]] = 0
    g = Group(gid=8, roles=[(0, 1, 1, 0), (1, 300, 2, 0)], pair=[[1, 0], [0, 1]], anchors=anchors)
    return bare_topo(free), build([g])


def many_used_pre(topo, gblob, exp=None):
    exp = ranked(topo, gblob) if exp is None else exp
    a, an = exp[0], exp[4]
    used = np.unique(a[1:][a[1:] >= 0])
    assert len(used) == 300 and a[0] == 650
    S = oracle_rows(topo, gblob)[0]
    alts = an[0][an[0] >= 0]
    assert len(alts) == 8 and (alts >= 300).all()
    late = [m for m in range(280, 300) if np.searchsorted(used, m) >= 256]
    assert late and all(S[m] > S[alts[0]] for m in late)
    return exp


def level_bitmap_levels(n):
    return [np.zeros(n, np.int32), ((np.arange(n) // 8) % 5).astype(np.int32)]


def lw_ranked_oracle(topo, gblob, rp, lvl):
    from test_gpu_lw_limits import oracle_lw
    return oracle_lw(topo, gblob, np.asarray(rp, np.int32).reshape(-1, 2), lvl, 8)


def level_bitmap_pre(topo, gblob, lvl):
    """The group took a level-1 domain, and B ranks nodes of it next to N's padding."""
    exp = lw_ranked_oracle(topo, gblob, [(1, -1)] * 3, lvl)
    assert topo.n % 4 != 0 or topo.n % 32 == 1
    assert exp[2][0] >= 0 and (exp[4][5] >= 0).any()
    assert (np.asarray(lvl[1])[exp[4][5][exp[4][5] >= 0]] == exp[2][0]).all()
    return exp


def coloc_pre(topo, gblob, rp, lvl):
    """Some pod has alternates, all inside its replica's level-1 domain."""
    exp = lw_ranked_oracle(topo, gblob, rp, lvl)
    a, an = exp[0], exp[4]
    dc = np.asarray(lvl[1])
    assert (an >= 0).any()
    for p in range(len(a)):
        x = an[p][an[p] >= 0]
        assert a[p] < 0 or (dc[x] == dc[a[p]]).all()
    return exp


# ---- 3. the committed replay across chunks

def slab_stride(n):
    lc = max(1, -(-n // 2048))
    chunk = min(2048, max(128, -(-(-(-n // lc)) // 128) * 128))
    return -(-(lc * chunk) // 32) * 32


def replay_chunks(gblob, assign, status, n):
    """The replay's chunks as the ranking builds them: per group not gang-failed, per wave with a placed replica, its
    role rows, a new chunk when they would pass max_rows.  Returns (chunks [[(g, wave)]], empty [(g, wave, chunk)])."""
    max_rows = max(8, REPLAY_FLOATS // slab_stride(n))
    chunks, empty, rowacc = [[]], [], 0
    for g, G in enumerate(wave_loop.groups_from_blob(gblob)):
        if status[g] == 2:
            continue
        s = wave_loop.GroupState(G)
        pod0 = int(np.asarray(gblob)[8 + 12 * g + 8])
        ord0 = np.concatenate([[0], np.cumsum(s.pending)])
        for w, wave in enumerate(s.waves):
            idx = [pod0 + ord0[ri] + o + c for ri, o, cnt in wave for c in range(cnt)]
            if not any(assign[i] >= 0 for i in idx):
                empty.append((g, w, len(chunks) - 1))
                continue
            if rowacc + len(wave) > max_rows:
                chunks.append([])
                rowacc = 0
            chunks[-1].append((g, w))
            rowacc += len(wave)
    return chunks, empty


CHUNK_GROUPS = 23
EMPTY_AT = (11, 3)      # (group, wave) with nothing placed, right where the first chunk ends
GANG_FAILED = 2


def chunk_case():
    """N = 1 638 400, 240 nodes with room 1..8, no other.  23 groups of 16 one-replica roles at levels 0..15 (16
    waves, every role paired with every other: a row's anchors are the group's earlier waves, `need` its unplaced
    roles); group 2 is a gang that cannot place (a role of demand 9), group 11's wave 3 places nothing (demand 9)
    and falls where the first chunk of 163 rows ends.  Replicas fill the best nodes in order, so later groups take
    the room the earlier groups' alternates had."""
    n = BITMAP_NODES
    rng = np.random.default_rng(77)
    free = np.zeros(n, np.int32)
    nodes = np.sort(rng.choice(np.arange(2, n), 239, replace=False))
    free[nodes] = rng.integers(1, 9, 239)
    free[n - 1] = 8
    groups = []
    for g in range(CHUNK_GROUPS):
        roles = [(L, 1, 9 if (g, L) == EMPTY_AT or (g == GANG_FAILED and L == 5) else 1, 0) for L in range(16)]
        groups.append(Group(gid=100 + g, roles=roles, pair=[[1] * 16 for _ in range(16)],
                            flags=STEP_GANG if g == GANG_FAILED else 0))
    return bare_topo(free), build(groups)


def chunk_pre(topo, gblob, a, s):
    """Chunks, the straddling group, the empty wave at the boundary, from the committed placements (a, s)."""
    chunks, empty = replay_chunks(gblob, a, s, topo.n)
    assert len(chunks) >= 2 and s[GANG_FAILED] == 2 and s[EMPTY_AT[0]] == 1
    where = {}
    for c, rows in enumerate(chunks):
        for g, w in rows:
            where.setdefault(g, set()).add(c)
    straddle = [g for g, cs in where.items() if len(cs) > 1]
    assert EMPTY_AT[0] in straddle
    g, w = EMPTY_AT
    before = max(c for gg, ww in [(g, v) for v in range(w)] for c, rows in enumerate(chunks) if (gg, ww) in rows)
    after = min(c for c, rows in enumerate(chunks) for gg, ww in rows if gg == g and ww > w)
    assert (g, w, before) in empty and after == before + 1
    return chunks, straddle


def chunk_removed(topo, gblob, a, chunks):
    """Alternates the groups ranked wholly in the first chunk have as a batch of their own that the full batch takes
    away, on nodes a group ranked wholly in later chunks placed on."""
    groups = wave_loop.groups_from_blob(gblob)
    first = {g for g, _ in chunks[0]}
    later = {g for c in chunks[1:] for g, _ in c} - first
    k = min(later)
    assert all(g < k for g in first - later) and first - {g for c in chunks[1:] for g, _ in c}
    prefix = [g for g in range(k) if g not in {g2 for c in chunks[1:] for g2, _ in c}]
    alone = cao.run_fleet_committed_ranked(topo, groups[:max(prefix) + 1], 8, fast=True)
    gb = np.asarray(gblob)
    used = np.bincount(a[a >= 0], minlength=topo.n)       # every replica of the case has demand 1
    taken = set()
    for g in later:
        p0, cnt = int(gb[8 + 12 * g + 8]), int(gb[8 + 12 * g + 9])
        taken |= set(a[p0:p0 + cnt][a[p0:p0 + cnt] >= 0].tolist())
    return {int(x) for x in alone[4].ravel() if x >= 0 and topo.free[x] - used[x] < 1} & taken


def committed_plain(topo, gblob):
    return co.result_arrays(co.run_fleet_committed(topo, wave_loop.groups_from_blob(gblob), fast=True))


# ---- 4. all eight levels

LEVEL_PAIRS = [(0, 7), (7, 0), (3, 5)]
LEVEL_GIDS = {7: 9, 0: 0, 1: (1 << 31) - 1, 2: 5, 3: 0, 4: 6, 5: 5, 6: 8}
LEVEL_ORDER = [7, 0, 1, 2, 3, 4, 5, 6]


def eight_levels(n=130):
    topo = synth.make_topology(n, seed=61, tiers=2, max_free=2)
    topo.domain_owner[:] = -1
    topo.free = np.full(n, 2, np.int32)
    r = np.random.default_rng(61).permutation(n)
    lv = np.stack([topo.domain, np.arange(n), np.arange(n) // 2, np.arange(n) // 4, r // 8, np.arange(n) // 16,
                   np.arange(n) // 32, np.arange(n) // 65]).astype(np.int32)
    nd = [int(x.max()) + 1 for x in lv]
    nd[0] = len(topo.domain_owner)
    occ = np.array([(5, 999, 1), (50, 999, 3), (20, 7777, 0), (40, 5, 2)], np.int32)   # level-7 domain 0 only
    return topo, lv, nd, occ


def level_groups(claims=()):
    """An exclusive group at every level (level 7 first), two pairs sharing gids, then idle groups with fixed domains
    (their claims): claims = [(level, fixed_domain, gid)]."""
    out = [Group(gid=LEVEL_GIDS[L], roles=[(0, 2, 1, ROLE_EXCLUSIVE), (0, 1, 1, 0)], pair=[[1, 1], [1, 1]],
                 flags=STEP_EXCLUSIVE, level=L) for L in LEVEL_ORDER]
    out += [Group(gid=gid, roles=[(0, 0, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE, fixed_domain=int(d),
                  level=L) for L, d, gid in claims]
    return out


def levels_dict(lv, nd, occ, gblob):
    import committed_levels_oracle as clo
    return dict(group_levels=clo.group_levels(gblob), level_domain=lv, owner=lo.derive_level_owner(lv, occ),
                n_domains=nd)


def eight_levels_case():
    """The batch without claims, then with a later claim at level b on the level-b domain of an alternate of the
    earlier group at level a, for every (a, b) of LEVEL_PAIRS."""
    topo, lv, nd, occ = eight_levels()
    base = build(level_groups())
    exp = cao.run_fleet_committed_ranked(topo, wave_loop.groups_from_blob(base), 8, fast=True,
                                         levels=levels_dict(lv, nd, occ, base))
    claims, picked = [], []
    for k, (La, Lb) in enumerate(LEVEL_PAIRS):
        g = LEVEL_ORDER.index(La)
        r = 3 * g                       # the group's first replica
        h = int(exp[4][r][0])
        assert h >= 0, (La, exp[4][r])
        claims.append((Lb, int(lv[Lb][h]), 20 + k))
        picked.append((r, h))
    return topo, lv, nd, occ, base, build(level_groups(claims)), picked


def eight_levels_pre(topo, lv, nd, occ, base, gblob, picked, exp=None):
    gb = np.asarray(gblob)
    lmask = 0
    for g in range(int(gb[2])):
        if gb[8 + 12 * g + 1] & STEP_EXCLUSIVE:
            lmask |= 1 << int(gb[8 + 12 * g + 10])
    assert lmask == 0xFF
    gids = {int(gb[8 + 12 * g]) for g in range(int(gb[2]))}
    assert {0, (1 << 31) - 1} <= gids
    exp = cao.run_fleet_committed_ranked(topo, wave_loop.groups_from_blob(gblob), 8, fast=True,
                                         levels=levels_dict(lv, nd, occ, gblob)) if exp is None else exp
    ng0 = len(LEVEL_ORDER)
    for r, h in picked:
        assert exp[0][r] >= 0 and h not in exp[4][r], (r, h, exp[4][r])
    assert (exp[1][ng0:] == 0).all()
    return exp


# ---- 5. the exactness bound of the ranking

def enumerated_bound(roles, pair, gang):
    """Per role, the largest need·8 + Σ_j pair·(replicas of j placed before the wave) of any wave it is in, over every
    vector of unplaced earlier replicas per role (none for a gang group)."""
    from test_gpu_lw_limits import enumerated_bound as pods_bound
    return pods_bound(roles, pair, [1] * len(roles), gang)


def exact_topo(n=130, seed=30, cap=24):
    topo = synth.make_topology(n, seed=seed, tiers=2, max_free=1)
    topo.domain_owner[:] = -1
    topo.free[:] = 0
    topo.free[np.random.default_rng(seed).choice(n, cap, replace=False)] = 1
    return topo


def anchor_limit(topo):
    import groups_gen as gg
    row_w = gg.wsum_max(topo) + 8000
    return ((1 << 24) + row_w - 1) // row_w


EXACT = [([[3]], (40,)), ([[1, 3], [7, 12]], (12, 20)), ([[3, 1, 12], [8, 1, 7], [1, 0, 1]], (4, 4, 9))]


def exact_case(i):
    """A non-gang group plus a last role with nothing pending whose pair column is 1 for every real role: c anchors
    on it raise every real role's anchor weight by c.  Returns (topo, blob(c), c at the bound, bound)."""
    from test_gpu_lw_limits import exact_group
    pair, pend = EXACT[i]
    topo = exact_topo()
    roles, full = exact_group(pair, pend)
    B = enumerated_bound(roles[:-1], [r[:-1] for r in full[:-1]], False)
    blob = lambda c: build([Group(gid=1, roles=roles, pair=full, anchors=[(7, len(pend), c)])])
    return topo, blob, anchor_limit(topo) - max(B), B


def exact_pre(i, topo, blob, c_at, B):
    if i == 0:   # wave 0 (32 replicas, room for 24) leaves the worst mix: 8 unplaced
        assert B == [3 * 24 + 16 * 8]
        a, s, _ = committed_plain(topo, blob(c_at - 1))
        assert (a[:32] >= 0).sum() == 24 and (a[32:40] < 0).all() and s.tolist() == [1]
