"""Oracle of leader-worker placement (rbgtopo_place_groups_lw, DESIGN.md §3.11; test infrastructure).

The §3.11 loop in numpy, read straight from the GROUPS blob and the (S, C) table.  Every wave is a step batch of the
oracle's own BLOB format (oracle/wave_loop.build_blob: role counts in pods, need over unplaced pods, one anchor per
placed pod, consumed capacity per node) scored by the CPU oracle (oracle/placer.py); its dense rows are all this file
takes from it.  Rule 3 is then restated literally: candidates with room, D* as §3.5 decides it, the level-C domains
enumerated with their pod capacity, the best one that holds the replica, the pods one after the other, and a replica
whose pods do not all fit reverted before the next one.  That enumeration costs O(N) per domain; `fast_domains()`
swaps in a one-pass form of the same choice (domain_fast) for fleets with one domain per node.
"""
from __future__ import annotations

import contextlib
import functools
from typing import List, Optional, Sequence

import numpy as np

from oracle import placer as oracle_placer
from oracle import wave_loop

HDR, GW = 8, 12
STEP_EXCLUSIVE, STEP_GANG, ROLE_EXCLUSIVE = 1, 2, 1
MAX_PODS, MAX_ROLES, NEED_CAP = 32, 8, 16


def best_node(mask: np.ndarray, row: np.ndarray) -> int:
    """The node of mask with the largest key(score, node): score descending, node ascending; -1 if none."""
    idx = np.flatnonzero(mask)
    if len(idx) == 0:
        return -1
    s = row[idx]
    return int(idx[s == s.max()][0])


def better(a: int, b: int, row: np.ndarray) -> bool:
    """key(row[a], a) > key(row[b], b); b = -1 loses."""
    return b < 0 or row[a] > row[b] or (row[a] == row[b] and a < b)


def pod_waves(pending: Sequence[int], levels: Sequence[int], S: Sequence[int]) -> List[List[tuple]]:
    """Waves of (role, first replica, replicas): one level at a time, <= 32 pods and <= 8 role rows, whole replicas."""
    waves: List[List[tuple]] = []
    cur: List[tuple] = []
    n = 0
    for ri in range(len(pending)):
        if cur and levels[ri] != levels[cur[-1][0]]:
            waves.append(cur)
            cur, n = [], 0
        left, first = int(pending[ri]), 0
        while left > 0:
            take = min(left, (MAX_PODS - n) // S[ri])
            if take == 0 or len(cur) == MAX_ROLES:
                waves.append(cur)
                cur, n = [], 0
                continue
            cur.append((ri, first, take))
            n += take * S[ri]
            left -= take
            first += take
    if cur:
        waves.append(cur)
    return waves


class LwGroup:
    def __init__(self, gb: np.ndarray, g: int, rp: np.ndarray, pod0: int):
        rec = gb[HDR + GW * g:HDR + GW * (g + 1)]
        self.gid, self.flags, self.fixed, q = int(rec[0]), int(rec[1]), int(rec[2]), int(rec[3])
        self.q = q
        rt = gb[rec[4]:rec[4] + 4 * q].reshape(q, 4)
        self.levels, self.pending = rt[:, 0].tolist(), rt[:, 1].tolist()
        self.demand, self.rflags = rt[:, 2].tolist(), rt[:, 3].tolist()
        self.pair = gb[rec[5]:rec[5] + q * q].reshape(q, q).astype(np.int64)
        self.S = [int(x) for x in rp[:, 0]]
        self.C = [int(x) for x in rp[:, 1]]
        self.anchors = {}
        for a in gb[rec[7]:rec[7] + 3 * rec[6]].reshape(-1, 3):
            k = (int(a[0]), int(a[1]))
            self.anchors[k] = self.anchors.get(k, 0) + int(a[2])
        self.consumed = {}
        self.unplaced = [p * s for p, s in zip(self.pending, self.S)]
        self.first_pod = list(np.concatenate([[0], np.cumsum(self.unplaced)[:-1]]).astype(int)) if q else []
        self.pod0 = pod0
        self.n_pods = sum(self.unplaced)
        self.waves = pod_waves(self.pending, self.levels, self.S)
        self.status, self.failed = 0, False

    def step(self, w: int) -> dict:
        roles, pair = [], []
        for ri, _, reps in self.waves[w]:
            need = min(NEED_CAP, sum(self.unplaced[q] for q in range(self.q) if self.pair[ri, q] > 0))
            roles.append((reps * self.S[ri], self.demand[ri], need, self.rflags[ri] & ROLE_EXCLUSIVE))
            pair.append([int(x) for x in self.pair[ri]])
        excl = bool(self.flags & STEP_EXCLUSIVE)
        return dict(gid=self.gid, flags=self.flags & (STEP_EXCLUSIVE | STEP_GANG),
                    fixed_domain=self.fixed if excl else -1, roles=roles, pair=pair,
                    anchors=[(n, q, c) for (n, q), c in sorted(self.anchors.items())],
                    consumed=sorted(self.consumed.items()))


def domain_literal(cand: np.ndarray, avail: np.ndarray, demand: int, S: int, dom: np.ndarray, row: np.ndarray) -> int:
    """D_r as rule 3 states it: enumerate the level-C domains of the candidates, count the pods each can hold, keep the
    best one that holds S (its best candidate by key); -1 if none.  O(N) per domain."""
    chosen, chosen_best = -1, -1
    for d in np.unique(dom[cand]):
        members = cand & (dom == d)
        cap = int((avail[members] // demand).sum()) if demand > 0 else S
        if cap < S:
            continue
        b = best_node(members, row)
        if better(b, chosen_best, row):
            chosen, chosen_best = int(d), b
    return chosen


def domain_fast(cand: np.ndarray, avail: np.ndarray, demand: int, S: int, dom: np.ndarray, row: np.ndarray) -> int:
    """domain_literal in one pass: per-domain pod capacity by bincount (S per candidate when demand = 0), then the best
    candidate among the domains that hold S.  O(N) per replica, so one domain per node stays cheap."""
    idx = np.flatnonzero(cand)
    if len(idx) == 0:
        return -1
    d = dom[idx]
    per = avail[idx] // demand if demand > 0 else np.full(len(idx), S, dtype=np.int64)
    cap = np.bincount(d, weights=per.astype(np.float64))   # sums below 2^53: exact
    keep = np.zeros(len(row), dtype=bool)
    keep[idx[cap[d] >= S]] = True
    b = best_node(keep, row)
    return int(dom[b]) if b >= 0 else -1


def place_wave(G: LwGroup, w: int, rows: np.ndarray, topo, excl_domain: np.ndarray, level_domain,
               choose=domain_literal) -> tuple:
    """Rule 3 for group G's wave w; rows[p] = the dense row of the wave's role p.  Returns (pods, status, D*).
    choose: how D_r is found (domain_literal or domain_fast; they agree)."""
    n = topo.n
    avail = topo.free.astype(np.int64).copy()
    for node, amt in G.consumed.items():
        avail[node] -= amt
    excl = bool(G.flags & STEP_EXCLUSIVE)
    dstar = -1
    if excl:
        if G.fixed >= 0:
            dstar = G.fixed
        else:
            for p, (ri, _, _) in enumerate(G.waves[w]):
                if G.rflags[ri] & ROLE_EXCLUSIVE:
                    b = best_node(rows[p] != -np.inf, rows[p])
                    dstar = int(excl_domain[b]) if b >= 0 else -1
                    break
    pods: List[int] = []
    unplaced = 0
    for p, (ri, _, reps) in enumerate(G.waves[w]):
        S, C, demand, row = G.S[ri], G.C[ri], G.demand[ri], rows[p]
        part = excl and bool(G.rflags[ri] & ROLE_EXCLUSIVE)
        scored = (row != -np.inf) & ((excl_domain == dstar) if part else True)
        for _ in range(reps):
            inside = np.ones(n, dtype=bool)
            ok = True
            if C >= 0:   # the best level-C domain that holds the replica
                dom = np.asarray(level_domain[C])
                chosen = choose(scored & (avail >= demand), avail, demand, S, dom, row)
                if chosen < 0:
                    ok = False
                else:
                    inside = dom == chosen
            picks: List[int] = []
            for _k in range(S if ok else 0):
                b = best_node(scored & inside & (avail >= demand), row)
                if b < 0:
                    ok = False
                    break
                avail[b] -= demand
                picks.append(b)
            if not ok:   # all or nothing: give the room back
                for b in picks:
                    avail[b] += demand
                picks = [-1] * S
                unplaced += 1
            pods.extend(picks)
    gang = bool(G.flags & STEP_GANG)
    if gang and unplaced:
        return [-1] * len(pods), 2, dstar
    return pods, 1 if unplaced else 0, dstar


_place_wave = place_wave   # the function itself, whatever the name place_wave is bound to


@contextlib.contextmanager
def fast_domains():
    """Inside the block place_wave finds D_r with domain_fast.  run_lw, lw_committed_oracle and lw_alternates_oracle
    all call place_wave through this module, so all three oracles then scale to one domain per node."""
    global place_wave
    saved = place_wave
    place_wave = functools.partial(_place_wave, choose=domain_fast)
    try:
        yield
    finally:
        place_wave = saved


def run_lw(topo, gblob, role_pods, level_domain=None, excl_domain=None, groups: Optional[Sequence[int]] = None):
    """The §3.11 loop.  topo: the snapshot the oracle scores (its domain / domain_owner decide feasibility);
    level_domain: the partitions a co-location level C indexes, row L = level L (default: [topo.domain]);
    excl_domain: the partition D* and the exclusive restriction read (default topo.domain);
    groups: the groups to place (default all; under snapshot semantics a group does not depend on the others).
    Returns (assign per pod of the whole blob, status[ng], domain[ng]); groups left out keep -1 / -9 / -9."""
    gb = np.asarray(gblob, dtype=np.int64)
    rp = np.asarray(role_pods, dtype=np.int64).reshape(-1, 2)
    ng = int(gb[2])
    level_domain = [topo.domain] if level_domain is None else level_domain
    excl_domain = np.asarray(topo.domain if excl_domain is None else excl_domain)
    G: List[LwGroup] = []
    r0 = pod0 = 0
    for g in range(ng):
        q = int(gb[HDR + GW * g + 3])
        G.append(LwGroup(gb, g, rp[r0:r0 + q], pod0))
        r0 += q
        pod0 += G[-1].n_pods
    assign = np.full(max(pod0, 0), -1, dtype=np.int32)
    status = np.full(ng, -9, dtype=np.int32)
    domain = np.full(ng, -9, dtype=np.int32)
    todo = list(range(ng)) if groups is None else list(groups)
    w = 0
    while True:
        active = [g for g in todo if not G[g].failed and w < len(G[g].waves)]
        if not active:
            break
        blob = wave_loop.build_blob([G[g].step(w) for g in active])
        r = oracle_placer.place(topo, blob, want_matrix=True, want_topk=False)
        if r["rc"] != 0:
            raise RuntimeError(f"oracle rc={r['rc']} in wave {w}")
        off = 0
        for g in active:
            X = G[g]
            rows, k = [], off
            for ri, _, reps in X.waves[w]:
                rows.append(r["matrix"][k])
                k += reps * X.S[ri]
            pods, st, dstar = place_wave(X, w, rows, topo, excl_domain, level_domain)
            off = k
            i, any_placed = 0, False
            for ri, first, reps in X.waves[w]:
                base = X.pod0 + X.first_pod[ri] + first * X.S[ri]
                for j in range(reps * X.S[ri]):
                    node = pods[i]
                    i += 1
                    assign[base + j] = node
                    if node >= 0:
                        any_placed = True
                        X.anchors[(node, ri)] = X.anchors.get((node, ri), 0) + 1
                        X.consumed[node] = X.consumed.get(node, 0) + X.demand[ri]
                        X.unplaced[ri] -= 1
            if (X.flags & STEP_EXCLUSIVE) and dstar >= 0 and any_placed:
                X.fixed = dstar
            X.status = max(X.status, st)
            if (X.flags & STEP_GANG) and st != 0:
                X.failed = True
        w += 1
    for g in todo:
        X = G[g]
        if X.failed:
            assign[X.pod0:X.pod0 + X.n_pods] = -1
            status[g], domain[g] = 2, -1
        else:
            status[g] = X.status
            domain[g] = X.fixed if X.flags & STEP_EXCLUSIVE else -1
    return assign, status, domain


def role_pods_for(gblob, fn) -> np.ndarray:
    """(S, C) per role of every group in blob order: fn(group, role) -> (S, C)."""
    gb = np.asarray(gblob, dtype=np.int64)
    out = []
    for g in range(int(gb[2])):
        for r in range(int(gb[HDR + GW * g + 3])):
            out.append(fn(g, r))
    return np.asarray(out, dtype=np.int32).reshape(-1, 2)

