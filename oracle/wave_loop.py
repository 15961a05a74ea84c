"""Oracle-side level / wave loop of whole RoleBasedGroups.  TEST INFRASTRUCTURE (same status as
oracle/placer.py): imported only by tests/, __graft_entry__.smoke() and bench.py's checker /
cpu_baseline / --impl reference legs.  Nothing here touches rbg_b200's native library: the
reference arm of bench.py builds its inputs with this file alone, so that the product `.so` is
never mapped into the reference process.

It restates, independently of rbg_b200/plugin.py and rbg_b200/blob.py:
  * the role order: dependency levels of `dependencyOrder` (pkg/dependency/dependency.go:129-205,
    via oracle/refpinned.dependency_order — names sorted, level = 1 + max(dep levels)), roles
    lexicographic inside a level, ordinals ascending (stateful_instance_set_utils.go:74-76);
  * the wave rule of DESIGN.md §3.2 (a wave = the next <= 32 replicas of <= 8 roles of one level);
  * the pair matrix (same role, dependency edge, shared CoordinatedPolicy rule) and
    need_rho = min(16, still-unplaced replicas of the paired roles);
  * the BLOB wire format of include/rbgtopo.h (one contiguous int32 array), and the GROUPS wire
    format it reads back (groups_from_blob: a raw GROUPS blob with explicit levels, pair weights and
    anchor counts runs through the same loop);
  * the feedback of a wave's placements into the next (anchors, consumed capacity, the fixed
    exclusive domain, gang all-or-nothing over the group: k8s-scheduler-plugin/manager.go:131).
Parity of the placements themselves is UNPINNED upstream (oracle/placer_oracle.c header).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import placer as oracle_placer
from . import refpinned

MAGIC, VERSION, HDR_WORDS, STEP_WORDS = 0x54474252, 1, 8, 16
STEP_EXCLUSIVE, STEP_GANG, ROLE_EXCLUSIVE = 1, 2, 1
MAX_STEP_ROLES, MAX_STEP_REPLICAS, NEED_CAP = 8, 32, 16


@dataclass
class ORole:
    name: str
    replicas: int
    deps: Sequence[str] = ()
    demand: int = 1
    exclusive: bool = True       # False = role-disable-exclusive (annotation.go:29)


@dataclass
class OGroup:
    name: str
    gid: int
    roles: List[ORole]
    rules: List[Sequence[str]] = field(default_factory=list)   # CoordinatedPolicy role sets
    exclusive: bool = False
    gang: bool = False
    placed: List[Tuple] = field(default_factory=list)   # (role, node) or (role, node, count) of scheduled pods
    fixed_domain: int = -1
    current: Dict[str, int] = field(default_factory=dict)         # replicas that already exist
    pair: Optional[Sequence[Sequence[int]]] = None   # explicit [Q][Q] weights instead of the host rule
    levels: Optional[Sequence[int]] = None           # explicit level per role: roles taken in the given order


def build_blob(steps: List[dict]) -> np.ndarray:
    """steps: dicts with gid, flags, fixed_domain, roles [(count, demand, need, role_flags)],
    pair [P][Q], anchors [(node, q, count)], consumed [(node, amount)]."""
    ns = len(steps)
    base = HDR_WORDS + ns * STEP_WORDS
    body: List[int] = []
    table = np.zeros((ns, STEP_WORDS), dtype=np.int64)
    racc = pacc = 0
    for i, s in enumerate(steps):
        P = len(s["roles"])
        Q = len(s["pair"][0]) if P and len(s["pair"][0]) else 0
        while (base + len(body)) & 3:
            body.append(0)
        role_off = base + len(body)
        for r in s["roles"]:
            body.extend(int(x) for x in r)
        pair_off = base + len(body)
        for row in s["pair"]:
            body.extend(int(x) for x in row)
        anchor_off = base + len(body)
        for a in s["anchors"]:
            body.extend(int(x) for x in a)
        cons_off = base + len(body)
        for c in s["consumed"]:
            body.extend(int(x) for x in c)
        R = sum(r[0] for r in s["roles"])
        table[i] = [s["gid"], s["flags"], s["fixed_domain"], P, role_off, Q, pair_off, len(s["anchors"]), anchor_off,
                    len(s["consumed"]), cons_off, R, racc, pacc, 0, 0]
        racc += R
        pacc += P
    words = base + len(body)
    out = np.zeros(words, dtype=np.int32)
    out[0:8] = [MAGIC, VERSION, ns, words, racc, pacc, 0, 0]
    out[HDR_WORDS:base] = table.reshape(-1)
    if body:
        out[base:] = np.asarray(body, dtype=np.int64)
    return out


class GroupState:
    """One group while its waves are placed."""

    def __init__(self, g: OGroup):
        self.g = g
        roles = g.roles
        self.Q = len(roles)
        index = {r.name: i for i, r in enumerate(roles)}
        if g.pair is not None:
            pair = np.asarray(g.pair, dtype=np.int64).reshape(self.Q, self.Q)
        else:
            pair = np.eye(self.Q, dtype=np.int64)
            for i, r in enumerate(roles):
                for d in r.deps:
                    pair[i, index[d]] = pair[index[d], i] = 1
            for rule in g.rules:
                ids = [index[x] for x in rule if x in index]
                for a in ids:
                    for b in ids:
                        pair[a, b] = 1
        self.pair = pair
        if g.levels is not None:               # consecutive roles of equal level form a level
            levels: List[List[str]] = []
            for i, r in enumerate(roles):
                if i == 0 or g.levels[i] != g.levels[i - 1]:
                    levels.append([])
                levels[-1].append(r.name)
        else:
            levels = refpinned.dependency_order({r.name: list(r.deps) for r in roles})
        self.first = [g.current.get(r.name, 0) for r in roles]
        self.pending = [max(r.replicas - g.current.get(r.name, 0), 0) for r in roles]
        self.unplaced = list(self.pending)
        self.anchors: Dict[Tuple[int, int], int] = {}
        for pod in g.placed:
            k = (int(pod[1]), index[pod[0]])
            self.anchors[k] = self.anchors.get(k, 0) + (int(pod[2]) if len(pod) > 2 else 1)
        self.consumed: Dict[int, int] = {}
        self.fixed_domain = g.fixed_domain
        self.failed = False
        self.status = 0
        self.nodes: Dict[str, int] = {}
        self.order: List[int] = []
        self.waves: List[List[Tuple[int, int, int]]] = []   # per wave: (role index, first ordinal, count)
        for level in levels:
            cur: List[Tuple[int, int, int]] = []
            n = 0
            for name in level:                 # dependency_order returns every level name-sorted
                ri = index[name]
                self.order.append(ri)
                left, ordinal = self.pending[ri], self.first[ri]
                while left > 0:
                    if n == MAX_STEP_REPLICAS or len(cur) == MAX_STEP_ROLES:
                        self.waves.append(cur)
                        cur, n = [], 0
                    take = min(left, MAX_STEP_REPLICAS - n)
                    cur.append((ri, ordinal, take))
                    n += take
                    left -= take
                    ordinal += take
            if cur:
                self.waves.append(cur)

    def step(self, w: int) -> dict:
        g = self.g
        roles, pair_rows = [], []
        for ri, _, cnt in self.waves[w]:
            need = min(NEED_CAP, sum(self.unplaced[q] for q in range(self.Q) if self.pair[ri, q] > 0))
            roles.append((cnt, g.roles[ri].demand, need, ROLE_EXCLUSIVE if g.roles[ri].exclusive else 0))
            pair_rows.append([int(x) for x in self.pair[ri]])
        return dict(gid=g.gid, flags=(STEP_EXCLUSIVE if g.exclusive else 0) | (STEP_GANG if g.gang else 0),
                    fixed_domain=self.fixed_domain if g.exclusive else -1, roles=roles, pair=pair_rows,
                    anchors=[(n, q, c) for (n, q), c in sorted(self.anchors.items())],
                    consumed=sorted(self.consumed.items()))

    def absorb(self, w: int, assign, status: int, domain: int) -> None:
        g = self.g
        k = 0
        for ri, ordinal, cnt in self.waves[w]:
            for c in range(cnt):
                node = int(assign[k])
                k += 1
                self.nodes[f"{g.name}-{g.roles[ri].name}-{ordinal + c}"] = node
                if node >= 0:
                    self.anchors[(node, ri)] = self.anchors.get((node, ri), 0) + 1
                    self.consumed[node] = self.consumed.get(node, 0) + g.roles[ri].demand
                    self.unplaced[ri] -= 1
        if g.exclusive and domain >= 0 and any(int(a) >= 0 for a in assign):
            self.fixed_domain = domain
        self.status = max(self.status, status)
        if g.gang and status != 0:
            self.failed = True

    def result(self) -> dict:
        nodes = {}
        for wave in self.waves:
            for ri, ordinal, cnt in wave:
                for c in range(cnt):
                    key = f"{self.g.name}-{self.g.roles[ri].name}-{ordinal + c}"
                    nodes[key] = -1 if self.failed else self.nodes.get(key, -1)
        if self.failed:
            return dict(status=2, nodes=nodes, domain=-1)
        return dict(status=self.status, nodes=nodes, domain=self.fixed_domain if self.g.exclusive else -1)

    def assign_in_group_order(self) -> List[int]:
        """Placements in the GROUPS-blob order: roles by (level, name), ordinals ascending."""
        res = self.result()["nodes"]
        out = []
        for ri in self.order:
            r = self.g.roles[ri]
            for c in range(self.pending[ri]):
                out.append(res[f"{self.g.name}-{r.name}-{self.first[ri] + c}"])
        return out


def run_fleet(topo, groups: Sequence[OGroup], nthreads: int = 1, want_matrix: bool = False,
              on_wave: Optional[Callable] = None, reuse_matrix: bool = False, want_topk: bool = False):
    """Level-synchronous wave loop over the CPU oracle.  Returns (states, blobs).
    on_wave(w, active_states, blob, oracle_result) is called after every wave (before absorb)."""
    states = [GroupState(g) for g in groups]
    blobs = []
    w = 0
    while True:
        active = [s for s in states if not s.failed and w < len(s.waves)]
        if not active:
            break
        blob = build_blob([s.step(w) for s in active])
        blobs.append(blob)
        r = oracle_placer.place(topo, blob, want_matrix=want_matrix, want_topk=want_topk, nthreads=nthreads,
                                reuse_matrix=reuse_matrix)
        if r["rc"] != 0:
            raise RuntimeError(f"oracle rc={r['rc']} in wave {w}")
        if on_wave is not None:
            on_wave(w, active, blob, r)
        off = 0
        for i, s in enumerate(active):
            cnt = sum(c for _, _, c in s.waves[w])
            s.absorb(w, r["assign"][off:off + cnt], int(r["status"][i]), int(r["domain"][i]))
            off += cnt
        w += 1
    return states, blobs


GROUPS_MAGIC, GROUP_WORDS = 0x47474252, 12


def groups_from_blob(gblob) -> List[OGroup]:
    """The groups of a GROUPS blob (include/rbgtopo.h, GROUPS section) as OGroups: roles in the blob's order with
    their levels, pending counts, demands and exclusive flags, the pair matrix as given, the anchors with their
    counts (repeated (node, role) records add up), the fixed domain and the gang / exclusive flags.  Role r of
    group i is named "r<r>" and its pending replicas get ordinals 0.., the group is named "g<i>"."""
    b = np.asarray(gblob, dtype=np.int64)
    if len(b) < HDR_WORDS or b[0] != GROUPS_MAGIC or b[1] != VERSION or b[3] != len(b):
        raise ValueError("not a GROUPS blob")
    out: List[OGroup] = []
    for i in range(int(b[2])):
        gid, flags, fixed, q, role_off, pair_off, na, anchor_off = (int(x) for x in b[HDR_WORDS + i * GROUP_WORDS:][:8])
        rt = b[role_off:role_off + 4 * q].reshape(q, 4)
        roles = [ORole(f"r{r}", int(rt[r, 1]), demand=int(rt[r, 2]), exclusive=bool(rt[r, 3] & ROLE_EXCLUSIVE))
                 for r in range(q)]
        pair = b[pair_off:pair_off + q * q].reshape(q, q).tolist()
        at = b[anchor_off:anchor_off + 3 * na].reshape(na, 3)
        placed = [(f"r{int(a[1])}", int(a[0]), int(a[2])) for a in at]
        out.append(OGroup(f"g{i}", gid, roles, exclusive=bool(flags & STEP_EXCLUSIVE), gang=bool(flags & STEP_GANG),
                          placed=placed, fixed_domain=fixed, pair=pair, levels=[int(x) for x in rt[:, 0]]))
    return out
