"""Oracle of exclusive topology at several levels (DESIGN.md §3.9; test infrastructure).

derive_level_owner   the owner vector of every level from the pod records, as §3.9 defines it (numpy);
derive_level_owner_fast  the same, vectorised (a million nodes x eight levels); the literal form stays the reference;
unused_gid           the smallest non-negative gid no group uses (the "other" owner of a level view);
constraining_gids    a restatement node by node: the set of exclusive groups whose pods constrain a labeled pod there;
owner_from_terms     the brute-force checker: the terms oracle.refpinned.exclusive_affinity_terms returns (the pinned
                     restatement of setExclusiveAffinities), evaluated with label-selector semantics on both sides of
                     every pair of pods;
group_view           the snapshot one group sees at level 0 in occupancy mode, in the form the existing oracle
                     takes (a per-domain owner map), so that oracle/wave_loop.py places the group unchanged.
"""
from __future__ import annotations

from typing import Sequence

import numpy as np

from oracle import refpinned
from rbg_b200 import synth

FREE, BLOCKED = -1, -2


def merge(a: int, b: int) -> int:
    if a == FREE:
        return b
    if b == FREE or a == b:
        return a
    return BLOCKED


def derive_level_owner(level_domain: np.ndarray, occ) -> np.ndarray:
    """level_domain[L][n] for L = 0..n_levels (row 0 = set_topology's domain); occ = (node, gid, level) records.
    Returns owner[L][n] with present_L / keyed_L / owner_L exactly as DESIGN.md §3.9 writes them."""
    dom = np.asarray(level_domain, dtype=np.int64)
    n_lv, n = dom.shape
    occ = np.asarray(occ, dtype=np.int64).reshape(-1, 3)
    present = [dict() for _ in range(n_lv)]
    keyed = [dict() for _ in range(n_lv)]
    for node, gid, lv in occ:
        for L in range(n_lv):
            d = int(dom[L, node])
            present[L][d] = merge(present[L].get(d, FREE), int(gid))
            if L == lv:
                keyed[L][d] = merge(keyed[L].get(d, FREE), int(gid))
    out = np.full((n_lv, n), FREE, dtype=np.int32)
    for v in range(n):
        k = FREE
        for L in range(n_lv):
            k = merge(k, keyed[L].get(int(dom[L, v]), FREE))
        for L in range(n_lv):
            out[L, v] = merge(present[L].get(int(dom[L, v]), FREE), k)
    return out


def merge_arrays(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """merge element by element."""
    return np.where(a == FREE, b, np.where((b == FREE) | (a == b), a, BLOCKED)).astype(np.int32)


def domain_owner_fast(dom: np.ndarray, nodes: np.ndarray, gids: np.ndarray) -> np.ndarray:
    """Per node v: the merge of the gids of the records (nodes[i], gids[i]) whose node shares v's domain — the one gid
    of a domain with one distinct gid, -2 with two or more, -1 with none.  Domains are renumbered densely first, so a
    partition with ~2^30 mostly empty domains costs O(n)."""
    ids, cd = np.unique(np.asarray(dom, dtype=np.int64), return_inverse=True)
    own = np.full(len(ids), FREE, dtype=np.int32)
    if len(nodes):
        pairs = np.unique(cd[nodes].astype(np.int64) << 32 | np.asarray(gids, dtype=np.int64))
        pd, pg = (pairs >> 32).astype(np.int64), (pairs & 0xFFFFFFFF).astype(np.int32)
        own[pd] = pg
        own[np.bincount(pd, minlength=len(ids)) >= 2] = BLOCKED
    return own[cd]


def derive_level_owner_fast(level_domain: np.ndarray, occ) -> np.ndarray:
    """derive_level_owner in vectorised numpy, for a million nodes x eight levels: per level, the distinct
    (domain, gid) pairs of the records (all of them for present_L, those of level L for keyed_L), then one gather per
    node."""
    dom = np.asarray(level_domain)
    n_lv, n = dom.shape
    occ = np.asarray(occ, dtype=np.int64).reshape(-1, 3)
    node, gid, lv = occ[:, 0], occ[:, 1], occ[:, 2]
    present = [domain_owner_fast(dom[L], node, gid) for L in range(n_lv)]
    k = np.full(n, FREE, dtype=np.int32)
    for L in range(n_lv):
        m = lv == L
        k = merge_arrays(k, domain_owner_fast(dom[L], node[m], gid[m]))
    return np.stack([merge_arrays(present[L], k) for L in range(n_lv)]) if n_lv else np.empty((0, n), np.int32)


def unused_gid(gids) -> int:
    """The smallest non-negative gid no group uses: an "other" owner that fits int32 even next to gid 2^31 - 1."""
    used = {int(g) for g in gids}
    return min(set(range(len(used) + 1)) - used)


def constraining_gids(level_domain: np.ndarray, occ, level: int, node: int) -> set:
    """Gids whose pods forbid a labeled pod of ANOTHER group, keyed at `level`, on `node` — the two required terms
    of the reference (pod_reconciler.go:172-231) evaluated pod by pod:
      * the incoming pod's own anti-affinity (key = `level`): every existing labeled pod in the same `level` domain;
      * an existing pod's anti-affinity (key = that pod's level), enforced symmetrically by kube-scheduler: every
        existing labeled pod in the same domain of ITS level.
    The incoming group's own affinity term is met by its own pods and by nothing else, so a node is usable by group g
    exactly when this set is empty or {g}; two or more gids block every group."""
    dom = np.asarray(level_domain)
    out = set()
    for nd, gid, lv in np.asarray(occ, dtype=np.int64).reshape(-1, 3):
        if dom[level, nd] == dom[level, node] or dom[lv, nd] == dom[lv, node]:
            out.add(int(gid))
    return out


def owner_from_sets(level_domain: np.ndarray, occ) -> np.ndarray:
    dom = np.asarray(level_domain)
    n_lv, n = dom.shape
    out = np.empty((n_lv, n), dtype=np.int32)
    for L in range(n_lv):
        for v in range(n):
            s = constraining_gids(dom, occ, L, v)
            out[L, v] = FREE if not s else (next(iter(s)) if len(s) == 1 else BLOCKED)
    return out


AFFINITY_KEY = "rbg.workloads.x-k8s.io/group-unique-hash"   # the label the terms select on (pod_reconciler.go:172-231)


def unique_key(gid: int) -> str:
    return f"hash-{gid}"


def selector_matches(expressions, labels: dict) -> bool:
    """metav1.LabelSelector matchExpressions (ANDed): In / NotIn / Exists / DoesNotExist."""
    for e in expressions:
        has = e["key"] in labels
        op = e["operator"]
        if op == "In" and not (has and labels[e["key"]] in e["values"]):
            return False
        if op == "NotIn" and has and labels[e["key"]] in e["values"]:
            return False
        if op == "Exists" and not has:
            return False
        if op == "DoesNotExist" and has:
            return False
    return True


def violates(level_domain: np.ndarray, keys, occ, gid: int, level: int, node: int) -> bool:
    """Does a labeled pod of exclusive group `gid`, whose annotation names keys[level], break a required
    anti-affinity term when bound on `node` next to the pods of `occ`?  Both directions: the incoming pod's own term
    against every existing pod, and every existing pod's term against the incoming pod (kube-scheduler enforces an
    existing pod's required anti-affinity symmetrically).  The affinity term is the group's own: it only decides which
    of the group's usable domains it must stay in (the fixed domain of §3.5), not who may use a node."""
    dom = np.asarray(level_domain)
    lv_of = {k: i for i, k in enumerate(keys)}
    mine = refpinned.exclusive_affinity_terms(unique_key(gid), keys[level], AFFINITY_KEY)["podAntiAffinity"]
    my_labels = {AFFINITY_KEY: unique_key(gid)}
    for nd, h, lv in np.asarray(occ, dtype=np.int64).reshape(-1, 3):
        theirs = refpinned.exclusive_affinity_terms(unique_key(int(h)), keys[int(lv)], AFFINITY_KEY)["podAntiAffinity"]
        L1 = lv_of[mine["topologyKey"]]
        if dom[L1, nd] == dom[L1, node] and selector_matches(mine["matchExpressions"], {AFFINITY_KEY: unique_key(int(h))}):
            return True
        L2 = lv_of[theirs["topologyKey"]]
        if dom[L2, nd] == dom[L2, node] and selector_matches(theirs["matchExpressions"], my_labels):
            return True
    return False


def owner_from_terms(level_domain: np.ndarray, occ, gids) -> np.ndarray:
    """owner[L][n] as the terms decide it for the groups `gids` (the gids of the records and at least one other):
    -1 when every group may use n at level L, g when only g may, -2 when none may."""
    dom = np.asarray(level_domain)
    n_lv, n = dom.shape
    keys = [f"example.com/level-{L}" for L in range(n_lv)]
    out = np.empty((n_lv, n), dtype=np.int32)
    for L in range(n_lv):
        for v in range(n):
            ok = [g for g in gids if not violates(dom, keys, occ, g, L, v)]
            out[L, v] = FREE if len(ok) == len(gids) else (ok[0] if len(ok) == 1 else BLOCKED)
    return out


def legacy_owner_map(domain: np.ndarray, n_domains: int, occ) -> np.ndarray:
    """The per-domain owner map level-0 records imply (-2 where two groups meet)."""
    owner = np.full(n_domains, FREE, dtype=np.int32)
    for node, gid, _ in np.asarray(occ, dtype=np.int64).reshape(-1, 3):
        d = int(domain[node])
        owner[d] = merge(int(owner[d]), int(gid))
    return owner


def group_view(topo: synth.Topology, owner0: np.ndarray, gid: int, other_gid: int) -> synth.Topology:
    """Level-0 snapshot of group `gid` as a per-domain owner map: domain' = 2·dom(n) + blocked(n) with
    owner'[2d] = -1 and owner'[2d + 1] = other_gid (!= gid).  Feasibility per node is that of owner0; D* (the domain
    of the best feasible node) is always even, so fixed' = 2·fixed and the reported domain is domain' // 2."""
    assert other_gid != gid
    blocked = ~((owner0 == FREE) | (owner0 == gid))
    dom = 2 * topo.domain.astype(np.int64) + blocked
    owner = np.full(2 * len(topo.domain_owner), FREE, dtype=np.int32)
    owner[1::2] = other_gid
    return synth.Topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free.copy(), dom.astype(np.int32), owner)


def groups_blob_for_view(gblob: np.ndarray, g: int) -> np.ndarray:
    """The blob with group g's fixed domain doubled (its numbering in group_view)."""
    b = np.array(gblob, dtype=np.int32, copy=True)
    off = 8 + 12 * g + 2
    if b[off] >= 0:
        b[off] *= 2
    return b


def random_levels(rng, n: int, domain: np.ndarray, n_levels: int, nested: Sequence[bool]):
    """Partitions of levels 1..n_levels: nested ones refine the level below (hostname-like when fine), the others
    are drawn independently."""
    rows = [np.asarray(domain, dtype=np.int32)]
    for L in range(1, n_levels + 1):
        k = int(rng.integers(1, max(2, n // 2) + 1))
        if nested[L - 1]:
            d = rows[-1].astype(np.int64) * k + rng.integers(0, k, n)
            _, d = np.unique(d, return_inverse=True)
        else:
            d = rng.integers(0, k, n)
            _, d = np.unique(d, return_inverse=True)
        rows.append(d.astype(np.int32))
    return np.stack(rows)


def random_occ(rng, n: int, n_levels: int, gids: Sequence[int], count: int) -> np.ndarray:
    return np.array([(int(rng.integers(0, n)), int(rng.choice(gids)), int(rng.integers(0, n_levels + 1)))
                     for _ in range(count)], dtype=np.int32).reshape(-1, 3)
