"""Seeded generator of irregular, valid cluster snapshots (test infrastructure, pure numpy).

`synth.make_topology` only builds near-uniform tiered clusters: an 8-node NVLink clique plus a few sampled peers per
tier, weights in {1, 10, 100, 1000}, free in 0..8, no isolated rows, no hubs.  The families here reach what the
snapshot refresh (k_base, the compact-key order sort, the incremental repair) handles beyond that:

  hubs      rows of degree 6 140-6 150 at every row_ptr & 3 alignment, among them the longest row k_base still stages
            (a segment of BASE_TILE_NNZ + 4 words) and one edge more (unstaged); a hub of degree >= 20 000
  sparse    N in {1, 2, 3, 127, 128, 129, 255, 257, 700}: isolated rows at 0, at N-1 and in runs longer than a
            256-row tile, single-edge components, weight-0 edges
  ties      every base equal (all weights 0, or a uniform ring) with free in {0, 8, 9, 32767} mixed in
  maxbase   one row attains (wsum_max + 8000) * 8, with bits(wsum_max * 8) < bits of that bound; and a snapshot whose
            largest base is 16 777 208, just under 2^24
  inexact   wsum_max * 8 >= 2^24 (accepted, need = 0 only); one of them sums to 2^28 in fp32 while its bound is 2^28 - 8
  large     N in {131 072, 131 073, 140 000}: both sides of k_base's fmin staging limit, 17 / 18 node bits

Every snapshot passes rbgtopo_set_topology's validation; all but the inexact ones keep wsum_max <= 60 000 so that steps
with need up to 16 and a few anchors stay inside the exactness bound.  `coverage()` reports which of the above a set of
cases reaches (tests/test_topo_gen.py)."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List

import numpy as np

from rbg_b200 import synth

F_CAP, SELF_W, MAX_FREE, MAX_W = 8, 8000, 32767, 65535
BASE_TILE_ROWS, BASE_TILE_NNZ, FMIN_SMEM_MAX = 256, 6144, 131072
SPARSE_SIZES = (1, 2, 3, 127, 128, 129, 255, 257, 700)
LARGE_SIZES = (131072, 131073, 140000)


@dataclass
class Case:
    name: str
    family: str
    topo: synth.Topology
    exact: bool          # (wsum_max + 8000) * 8 < 2^24: base is exact and need >= 1 steps are admitted


def from_edges(n: int, u, v, w, free, owned_frac: float = 0.0, seed: int = 0) -> synth.Topology:
    """Symmetric CSR from undirected edges (u != v; a repeated pair keeps its first weight), domains of 8 nodes."""
    u = np.asarray(u, dtype=np.int64)
    v = np.asarray(v, dtype=np.int64)
    w = np.asarray(w, dtype=np.int64)
    assert (u != v).all() and ((w >= 0) & (w <= MAX_W)).all()
    lo, hi = np.minimum(u, v), np.maximum(u, v)
    _, first = np.unique(lo * n + hi, return_index=True)
    lo, hi, w = lo[first], hi[first], w[first]
    a = np.concatenate([lo, hi])
    b = np.concatenate([hi, lo])
    ww = np.concatenate([w, w])
    o = np.lexsort((b, a))
    a, b, ww = a[o], b[o], ww[o]
    row_ptr = np.zeros(n + 1, dtype=np.int64)
    np.add.at(row_ptr, a + 1, 1)
    row_ptr = np.cumsum(row_ptr)
    domain = (np.arange(n) // 8).astype(np.int32)
    owner = np.full(int(domain.max()) + 1, -1, dtype=np.int32)
    if owned_frac > 0:
        rng = np.random.default_rng(seed + 7)
        owner[rng.random(len(owner)) < owned_frac] = 1_000_000
    return synth.Topology(row_ptr.astype(np.int32), b.astype(np.int32), ww.astype(np.int32),
                          np.asarray(free, dtype=np.int32).copy(), domain, owner)


def edges_of(topo):
    """(u, v, w) of every undirected edge, u < v."""
    rows = np.repeat(np.arange(topo.n), np.diff(topo.row_ptr))
    keep = rows < topo.col_idx
    return rows[keep], topo.col_idx[keep].astype(np.int64), topo.edge_w[keep].astype(np.int64)


# ---------------------------------------------------------------- plain exact references
def wsum_rows(topo) -> np.ndarray:
    cs = np.concatenate([[0], np.cumsum(topo.edge_w, dtype=np.int64)])
    return cs[topo.row_ptr[1:]] - cs[topo.row_ptr[:-1]]


def wsum_max(topo) -> int:
    return int(wsum_rows(topo).max()) if topo.n else 0


def base_int(topo, free=None) -> np.ndarray:
    """base = Σ w·min(free[col], 8) + 8000·min(free, 8), in int64."""
    fm = np.minimum(np.asarray(topo.free if free is None else free, dtype=np.int64), F_CAP)
    terms = topo.edge_w.astype(np.int64) * fm[topo.col_idx]
    cs = np.concatenate([[0], np.cumsum(terms)])
    return cs[topo.row_ptr[1:]] - cs[topo.row_ptr[:-1]] + SELF_W * fm


def base_ref(topo, free=None) -> np.ndarray:
    return base_int(topo, free).astype(np.float32)


def orderable_u32(x: np.ndarray) -> np.ndarray:
    b = np.asarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return np.where(b >> np.uint64(31), b ^ np.uint64(0xFFFFFFFF), b ^ np.uint64(0x80000000))


def keys_of(base: np.ndarray, nodes: np.ndarray) -> np.ndarray:
    """key(base, node) = (orderable_u32(base) << 32) | (0xFFFFFFFF - node), the form the library stores."""
    return (orderable_u32(base) << np.uint64(32)) | (np.uint64(0xFFFFFFFF) - np.asarray(nodes, dtype=np.uint64))


def order_ref(base: np.ndarray, lo: int = 0, hi: int = -1) -> np.ndarray:
    """Nodes [lo, hi) by (base desc, node asc) as keys: descending key order."""
    hi = len(base) if hi < 0 else hi
    k = keys_of(base[lo:hi], np.arange(lo, hi))
    return np.sort(k)[::-1]


def key_node(keys: np.ndarray) -> np.ndarray:
    return (np.uint64(0xFFFFFFFF) - (keys & np.uint64(0xFFFFFFFF))).astype(np.int64)


def pos_ref(order: np.ndarray) -> np.ndarray:
    pos = np.full(len(order), -1, dtype=np.int32)
    pos[key_node(order)] = np.arange(len(order), dtype=np.int32)
    return pos


def base_tiles(row_ptr) -> List[tuple]:
    """k_base's tiles as rbgtopo_set_topology builds them: (r0, r1) with r1 - r0 <= 256 rows and a 16-byte aligned
    segment of <= BASE_TILE_NNZ words, an over-long row alone."""
    rp = np.asarray(row_ptr, dtype=np.int64)
    n = len(rp) - 1
    out, r = [], 0
    while r < n:
        a0 = int(rp[r]) & ~3
        r1 = r
        while r1 < n and r1 - r < BASE_TILE_ROWS and rp[r1 + 1] - a0 <= BASE_TILE_NNZ:
            r1 += 1
        if r1 == r:
            r1 = r + 1
        out.append((r, r1))
        r = r1
    return out


def segment(row_ptr, r0: int, r1: int) -> int:
    """Words k_base stages for tile (r0, r1): staged while <= BASE_TILE_NNZ + 4."""
    return int(row_ptr[r1]) - (int(row_ptr[r0]) & ~3)


# ---------------------------------------------------------------- families
def _body(rng, n: int, deg: int, wmax: int):
    """A sparse random body: ~deg random edges per node, weights 1..wmax."""
    m = n * deg // 2
    u = rng.integers(0, n, size=m)
    v = rng.integers(0, n, size=m)
    keep = u != v
    return u[keep], v[keep], rng.integers(1, wmax + 1, size=int(keep.sum()))


def hubs(seed: int = 0) -> synth.Topology:
    """8 hubs of degree 6 140-6 150 among 7 000 nodes; (degree, row_ptr & 3) per hub chosen so that the single-row tiles
    have segments 6 140 .. 6 152, incl. exactly BASE_TILE_NNZ + 4 (staged) and BASE_TILE_NNZ + 5 (unstaged)."""
    rng = np.random.default_rng(seed)
    n = 7000
    plan = [(6140, 0), (6144, 1), (6145, 3), (6146, 3), (6147, 2), (6150, 2), (6148, 0), (6141, 1)]
    hub_nodes = np.array([400 + 800 * i for i in range(len(plan))])
    is_hub = np.zeros(n, dtype=bool)
    is_hub[hub_nodes] = True
    others = np.nonzero(~is_hub)[0]
    bu, bv, bw = _body(rng, n, 3, 1000)
    keep = ~is_hub[bu] & ~is_hub[bv]
    U, V, W = [bu[keep]], [bv[keep]], [bw[keep]]
    for h, (deg, _) in zip(hub_nodes, plan):
        nb = rng.choice(others, size=deg, replace=False)
        U.append(np.full(deg, h)); V.append(nb); W.append(rng.integers(1, 10, size=deg))
    free = rng.integers(0, 13, size=n)
    free[hub_nodes] = rng.integers(1, 13, size=len(hub_nodes))
    topo = from_edges(n, np.concatenate(U), np.concatenate(V), np.concatenate(W), free, owned_frac=0.1, seed=seed)
    # align every hub: single-edge links between non-hub nodes either side of the hub shift row_ptr[hub] by one
    u, v, w = edges_of(topo)
    U, V, W = [u], [v], [w]
    for h, (_, off) in zip(hub_nodes, plan):
        topo = from_edges(n, np.concatenate(U), np.concatenate(V), np.concatenate(W), free, owned_frac=0.1, seed=seed)
        d = (off - int(topo.row_ptr[h])) % 4
        adj = set(topo.col_idx[topo.row_ptr[h - 3]:topo.row_ptr[h - 2]].tolist())
        cand = [x for x in range(h + 1, h + 200) if not is_hub[x] and x not in adj][:d]
        U.append(np.full(d, h - 3)); V.append(np.array(cand, dtype=np.int64)); W.append(np.full(d, 5))
    topo = from_edges(n, np.concatenate(U), np.concatenate(V), np.concatenate(W), free, owned_frac=0.1, seed=seed)
    for h in hub_nodes:   # the last edge of every hub row counts in base (the tail lane of k_base)
        topo.free[topo.col_idx[topo.row_ptr[h + 1] - 1]] = 6
    return topo


def big_hub(seed: int = 0) -> synth.Topology:
    """One hub of degree 20 000 in a 24 000-node tiered cluster (weights 1 / 2 on the hub)."""
    rng = np.random.default_rng(seed)
    n = 24000
    base = synth.make_topology(n, seed=seed + 3, tiers=3)
    u, v, w = edges_of(base)
    h = 11111
    nb = rng.choice(np.delete(np.arange(n), h), size=20000, replace=False)
    topo = from_edges(n, np.concatenate([np.full(20000, h), u]), np.concatenate([nb, v]),
                      np.concatenate([rng.integers(1, 3, size=20000), w]), rng.integers(0, 11, size=n))
    return topo


def sparse(n: int, seed: int = 0) -> synth.Topology:
    """Isolated rows at 0 and N-1 (and [100, 400) when N >= 700), single-edge components with weights 0 .. 50 000,
    a few short paths; everything else isolated."""
    rng = np.random.default_rng(seed + n)
    iso = np.zeros(n, dtype=bool)
    iso[0] = iso[n - 1] = True
    if n >= 700:
        iso[100:400] = True
    live = np.nonzero(~iso)[0]
    rng.shuffle(live)
    U, V, W = [], [], []
    npairs = len(live) // 3
    for i in range(npairs):                       # single-edge components
        U.append(live[2 * i]); V.append(live[2 * i + 1]); W.append(int(rng.choice([0, 0, 1, 7, 1000, 50000])))
    rest = live[2 * npairs:]
    for a, b in zip(rest[:-1], rest[1:]):          # one path through the rest, some of it weight 0
        if rng.random() < 0.7:
            U.append(a); V.append(b); W.append(int(rng.choice([0, 3, 100])))
    free = rng.integers(0, 13, size=n)
    free[rng.random(n) < 0.1] = int(rng.choice([9, 30, MAX_FREE]))
    return from_edges(n, np.array(U, dtype=np.int64), np.array(V, dtype=np.int64), np.array(W, dtype=np.int64), free)


def ties(n: int, variant: str, seed: int = 0) -> synth.Topology:
    """"zero": a ring of weight-0 edges, free in {0, 8, 9, 32767} (two base values over the whole snapshot);
    "ring": a ring of weight 1000, free in {8, 9, 32767} (one base value: the order is node-ascending)."""
    rng = np.random.default_rng(seed + n)
    u = np.arange(n)
    v = (u + 1) % n
    keep = u != v
    if variant == "zero":
        w = np.zeros(n, dtype=np.int64)
        free = rng.choice([0, 8, 9, MAX_FREE], size=n)
    else:
        w = np.full(n, 1000, dtype=np.int64)
        free = rng.choice([8, 9, MAX_FREE], size=n)
    if n == 2:                                     # (0, 1) and (1, 0) are one edge
        keep[1] = False
    return from_edges(n, u[keep], v[keep], w[keep], free)


def max_base(wsum_top: int, n: int = 600, seed: int = 0, wcap: int = 1000) -> synth.Topology:
    """Node 5 has edge weights summing to wsum_top (each <= wcap) and it and its neighbourhood have free >= 8: its base
    is exactly (wsum_top + 8000) * 8, the bound the compact sort key reserves bits for.  Every other row sums to less."""
    rng = np.random.default_rng(seed)
    k = -(-wsum_top // wcap)
    ws = np.full(k, wcap, dtype=np.int64)
    ws[-1] = wsum_top - wcap * (k - 1)
    hub = 5
    nb = rng.choice(np.arange(10, n), size=k, replace=False)
    bu, bv, bw = _body(rng, n, 2, 20)
    keep = (bu != hub) & (bv != hub) & ~np.isin(bu, nb) & ~np.isin(bv, nb)
    free = rng.integers(0, 13, size=n)
    free[nb] = rng.choice([8, 9, 40, MAX_FREE], size=k)
    free[hub] = 8
    topo = from_edges(n, np.concatenate([np.full(k, hub), bu[keep]]), np.concatenate([nb, bv[keep]]),
                      np.concatenate([ws, bw[keep]]), free)
    assert wsum_max(topo) == wsum_top and int(base_int(topo).max()) == (wsum_top + SELF_W) * F_CAP
    return topo


def inexact(deg: int, last_w: int, n: int = 800, seed: int = 0) -> synth.Topology:
    """Node 3 has deg - 1 edges of weight 65 535 and one of weight last_w, all neighbours free >= 8."""
    rng = np.random.default_rng(seed)
    hub = 3
    nb = rng.choice(np.arange(10, n), size=deg, replace=False)
    ws = np.full(deg, MAX_W, dtype=np.int64)
    ws[-1] = last_w
    bu, bv, bw = _body(rng, n, 2, 1000)
    keep = (bu != hub) & (bv != hub)
    free = rng.integers(0, 13, size=n)
    free[nb] = rng.choice([8, 12, MAX_FREE], size=deg)
    free[hub] = 9
    return from_edges(n, np.concatenate([np.full(deg, hub), bu[keep]]), np.concatenate([nb, bv[keep]]),
                      np.concatenate([ws, bw[keep]]), free)


def large(n: int, seed: int = 0) -> synth.Topology:
    """A 3-tier synth cluster with four hubs of degree 3 000 (weights 1..9)."""
    rng = np.random.default_rng(seed + n)
    base = synth.make_topology(n, seed=seed + n, tiers=3)
    u, v, w = edges_of(base)
    U, V, W = [u], [v], [w]
    for h in (0, n // 3, n // 2 + 1, n - 1):
        nb = rng.choice(n, size=3000, replace=False)
        nb = nb[nb != h]
        U.append(np.full(len(nb), h)); V.append(nb); W.append(rng.integers(1, 10, size=len(nb)))
    free = rng.integers(0, 13, size=n)
    return from_edges(n, np.concatenate(U), np.concatenate(V), np.concatenate(W), free, owned_frac=0.05, seed=seed)


def exact_snapshot(topo) -> bool:
    return (wsum_max(topo) + SELF_W) * F_CAP < (1 << 24)


def _case(name, family, topo) -> Case:
    return Case(name, family, topo, exact_snapshot(topo))


# (name, family, builder): the seed set of tests/test_gpu_snapshot.py
BUILDERS = {
    "hubs": ("hubs", lambda: hubs(1)),
    "big_hub": ("hubs", lambda: big_hub(2)),
    **{f"sparse_{n}": ("sparse", (lambda n=n: lambda: sparse(n, 3))()) for n in SPARSE_SIZES},
    "ties_zero": ("ties", lambda: ties(20000, "zero", 4)),
    "ties_ring": ("ties", lambda: ties(20000, "ring", 5)),
    "ties_ring_3": ("ties", lambda: ties(3, "ring", 6)),
    "maxbase_bits": ("maxbase", lambda: max_base(30000, seed=7)),          # bits(240 000) = 18 < bits(304 000) = 19
    "maxbase_2p24": ("maxbase", lambda: max_base(2089151, seed=8, wcap=MAX_W)),   # largest base 16 777 208
    "inexact_40": ("inexact", lambda: inexact(40, MAX_W, seed=9)),
    "inexact_2p28": ("inexact", lambda: inexact(512, 58046, seed=10)),   # bound 2^28 - 8, fp32 sum 2^28
    **{f"large_{n}": ("large", (lambda n=n: lambda: large(n, 11))()) for n in LARGE_SIZES},
}
NAMES = list(BUILDERS)
_CACHE: Dict[str, Case] = {}


def make(name: str) -> Case:
    """The named case (cached: the large ones take a second to build).  Callers that modify the topology copy it."""
    if name not in _CACHE:
        fam, fn = BUILDERS[name]
        _CACHE[name] = _case(name, fam, fn())
    return _CACHE[name]


def copy_topo(t: synth.Topology) -> synth.Topology:
    return synth.Topology(t.row_ptr.copy(), t.col_idx.copy(), t.edge_w.copy(), t.free.copy(), t.domain.copy(),
                          t.domain_owner.copy())


def k_base_fp32(topo, r: int) -> np.float32:
    """base[r] as k_base sums it in fp32: 8 lanes over the row's edges (lane s takes edge rb + s, rb + s + 8, ...), a
    shuffle butterfly over lane distances 4, 2, 1, then the self term.  Differs from base_ref only past 2^24."""
    fm = np.minimum(topo.free.astype(np.int64), F_CAP)
    rb, re = int(topo.row_ptr[r]), int(topo.row_ptr[r + 1])
    lanes = []
    for s in range(8):
        acc = np.float32(0)
        for j in range(rb + s, re, 8):
            acc = np.float32(acc + np.float32(topo.edge_w[j]) * np.float32(fm[topo.col_idx[j]]))
        lanes.append(acc)
    for d in (4, 2, 1):
        lanes = [np.float32(lanes[s] + lanes[s ^ d]) for s in range(8)]
    return np.float32(lanes[0] + np.float32(SELF_W) * np.float32(fm[r]))


BULLETS = ("hub_align_0", "hub_align_1", "hub_align_2", "hub_align_3", "hub_staged_max", "hub_unstaged_min", "hub_20000",
           *[f"sparse_n{n}" for n in SPARSE_SIZES], "isolated_first", "isolated_last", "isolated_run_gt256",
           "single_edge_component", "zero_weight_edge", "ties_all_equal", "ties_zero_weights",
           "free_0", "free_8", "free_9", "free_32767", "max_base_all_bits", "max_base_2p24", "inexact",
           "inexact_rounds_past_bound", *[f"large_n{n}" for n in LARGE_SIZES], "fmin_not_staged")


def _bits(x: int) -> int:
    return max(1, int(x).bit_length())


def coverage(case: Case) -> Dict[str, bool]:
    c = dict.fromkeys(BULLETS, False)
    t = case.topo
    n = t.n
    deg = np.diff(t.row_ptr)
    for r0, r1 in base_tiles(t.row_ptr):
        if r1 - r0 == 1 and 6140 <= deg[r0] <= 6150:
            c[f"hub_align_{int(t.row_ptr[r0]) & 3}"] = True
        if r1 - r0 == 1 and deg[r0] > 0:
            seg = segment(t.row_ptr, r0, r1)
            c["hub_staged_max"] |= seg == BASE_TILE_NNZ + 4
            c["hub_unstaged_min"] |= seg == BASE_TILE_NNZ + 5
    c["hub_20000"] = bool((deg >= 20000).any())
    if case.family == "sparse":
        c[f"sparse_n{n}"] = True
    iso = deg == 0
    c["isolated_first"] = bool(iso[0]) and n > 1
    c["isolated_last"] = bool(iso[-1]) and n > 1
    run = best = 0
    for x in iso:
        run = run + 1 if x else 0
        best = max(best, run)
    c["isolated_run_gt256"] = best > BASE_TILE_ROWS and best < n
    u, v, w = edges_of(t)
    c["single_edge_component"] = bool(((deg[u] == 1) & (deg[v] == 1)).any())
    c["zero_weight_edge"] = bool((w == 0).any())
    if case.exact:
        b = base_int(t)
        c["ties_all_equal"] = n > 100 and len(np.unique(b)) == 1
    c["ties_zero_weights"] = len(w) > 0 and not w.any() and n > 100
    for f in (0, 8, 9, MAX_FREE):
        c[f"free_{f}"] = bool((t.free == f).any())
    ws = wsum_max(t)
    bound = (ws + SELF_W) * F_CAP
    if case.exact:
        c["max_base_all_bits"] = _bits(ws * F_CAP) < _bits(bound) and int(base_int(t).max()) == bound
        c["max_base_2p24"] = int(base_int(t).max()) == 16777208
    else:
        c["inexact"] = True
        hub = int(np.argmax(wsum_rows(t)))
        c["inexact_rounds_past_bound"] = _bits(int(k_base_fp32(t, hub))) > _bits(bound)
    if case.family == "large":
        c[f"large_n{n}"] = True
    c["fmin_not_staged"] = n > FMIN_SMEM_MAX
    return c
