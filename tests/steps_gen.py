"""Seeded generator of step-level BLOB batches at the limits of the ABI (test infrastructure).

The step batches of the parity tests (test_gpu_parity._random_steps, test_gpu_snapshot._steps) stay far inside what
include/rbgtopo.h admits: <= 5 roles per step, Q <= 7, pair weights 0-2, anchor counts 1-2, consumed amounts 1-3,
synth topologies only.  `make_case(seed, n_nodes, n_steps)` builds a snapshot and a BLOB batch that reach the limits
instead: 8-role steps of 32 replicas (the 256-thread selection CTA, rows 5-7 of k_score_emit's role table), one-role
steps of 32, Q = 16 (pair-matrix columns 8-15) and Q = 0, need 0 and 16 independent of the counts, asymmetric pair
weights to 5, all-zero pair rows, anchor counts 0 and > 1 in repeated records, anchors on full nodes, on a hub and on
isolated nodes, consumed amounts 0 and 32 767, duplicated consumed nodes whose amounts sum past free, consumed nodes
that are anchors too, steps on both sides of k_score_emit's two-record branch in one launch, the exclusive corners
(fixed domains on non-exclusive steps and owned by other gids, every role opted out, a first participating role other
than role 0 or infeasible everywhere, self-owned domains, repeated gids), gang steps that fail and non-gang steps that
place part of their replicas.  `coverage()` reports which of those (BULLETS) a set of cases reached, so a test can
assert that its seeds still reach every one.

Every step stays under the exactness bound the way validate_blob checks it: need·8 + Σ pair·count of every role, all
anchors counted on one node, below ceil(2^24 / (wsum_max + 8000)) (`exact_ok`)."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List

import numpy as np

import topo_gen as tg
from rbg_b200 import synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, STEP_GANG, BlobBuilder, Step

MAX_STEP_ROLES, MAX_STEP_REPLICAS, MAX_Q, NEED_CAP, F_CAP, SELF_W, MAX_FREE, KS = 8, 32, 16, 16, 8, 8000, 32767, 32
FOREIGN_GID = 1_000_000          # owner of the domains topo_gen.from_edges marks as owned

# The seed set of the GPU parity tests: (seed, nodes, steps).  N < 32 gives K > N; N % 4 != 0 runs the tail mask of the
# last float4 group; N = 1 and 3 have no background list left once the patched nodes are taken out.  17 and 33 steps
# leave a short last block of k_score_emit's 4-step blocks, 4 fills one exactly, 5 leaves a single step.
# tests/test_steps_gen.py asserts that together they reach every entry of BULLETS.
CASES = [(1, 1, 5), (2, 3, 4), (3, 7, 17), (4, 31, 33), (5, 33, 17), (6, 130, 33), (7, 2049, 17), (8, 4097, 33),
         (9, 130, 1), (10, 2049, 5)]

KINDS = ("wide", "single", "free", "exclusive", "consumed", "fixed_plain")


@dataclass
class Case:
    topo: synth.Topology
    steps: List[Step]
    blob: np.ndarray
    hubs: List[int]
    isolated: List[int]


def amax_limit(topo) -> int:
    """validate_blob's bound: a role is admitted while need·8 + Σ pair·count < ceil(2^24 / (wsum_max + 8000))."""
    return -(-(1 << 24) // (tg.wsum_max(topo) + SELF_W))


def role_mass(step: Step, p: int) -> int:
    return step.roles[p][2] * F_CAP + sum(step.pair[p][q] * c for _, q, c in step.anchors)


def exact_ok(step: Step, limit: int) -> bool:
    return all(role_mass(step, p) < limit for p in range(len(step.roles)))


def patch_capacity(topo, step: Step) -> int:
    """validate_blob's per-step patch capacity: consumed records + the closed neighbourhood of every anchor record."""
    deg = np.diff(topo.row_ptr)
    return len(step.consumed) + sum(int(deg[a[0]]) + 1 for a in step.anchors)


def topology(seed: int, n: int) -> tuple:
    """A synth cluster (NVLink cliques of 8 + sampled peers) with, from N = 7 up, one hub linked to a quarter of the
    nodes (weights 1-3) and two isolated nodes, the last node one of them; 30 % of the nodes full, a few with free 9 or
    12, 30 % of the domains owned by a foreign gid from N = 16 up.  Returns (topo, hubs, isolated)."""
    rng = np.random.default_rng(seed)
    base = synth.make_topology(n, seed=seed, tiers=2 if n < 256 else 3, max_free=4)
    u, v, w = tg.edges_of(base)
    hubs: List[int] = []
    if n >= 7:
        iso = sorted({n - 1, int(rng.integers(1, n - 1))})
        hub = next(x for x in rng.permutation(n).tolist() if x not in iso)
        keep = ~np.isin(u, iso) & ~np.isin(v, iso)
        others = np.array([x for x in range(n) if x != hub and x not in iso])
        k = max(3, min(len(others), n // 4))
        nb = rng.choice(others, size=k, replace=False)
        u = np.concatenate([u[keep], np.full(k, hub)])
        v = np.concatenate([v[keep], nb])
        w = np.concatenate([w[keep], rng.integers(1, 4, size=k)])
        hubs = [hub]
    free = base.free.astype(np.int64)
    free[rng.random(n) < 0.3] = 0
    free[rng.random(n) < 0.05] = int(rng.choice([9, 12]))
    topo = tg.from_edges(n, u, v, w, free, owned_frac=0.3 if n >= 16 else 0.0, seed=seed)
    iso = np.nonzero(np.diff(topo.row_ptr) == 0)[0].tolist()
    return topo, hubs, iso


def _counts(rng, P: int, R: int) -> List[int]:
    return (rng.multinomial(R - P, np.ones(P) / P) + 1).tolist()


def _lower_to_bound(step: Step, limit: int) -> None:
    """Lower the heaviest pair weight of a role (its need once the row is zero) until the role is under the bound."""
    pair = [list(r) for r in step.pair]
    roles = [list(r) for r in step.roles]
    step.pair, step.roles = pair, roles
    for p in range(len(roles)):
        while role_mass(step, p) >= limit:
            if any(pair[p]):
                pair[p][int(np.argmax(pair[p]))] -= 1
            else:
                roles[p][2] -= 1
    step.roles = [tuple(r) for r in roles]


def _step(rng, kind: str, topo, hubs: List[int], iso: List[int], limit: int) -> Step:
    n = topo.n
    full = np.nonzero(topo.free == 0)[0].tolist()
    demand_big = int(topo.free.max()) + 1                      # fits no node
    if kind == "wide":
        P, R = 8, 32
    elif kind == "single":
        P, R = 1, 32
    elif kind == "exclusive":
        P = int(rng.integers(2, 9))
        R = int(rng.integers(P, 33))
    else:
        P = int(rng.integers(1, 9))
        R = int(rng.integers(P, 33))
    counts = _counts(rng, P, R)
    Q = {"wide": 16, "single": int(rng.choice([1, 16])), "consumed": 0, "exclusive": int(rng.choice([P, 16])),
         "fixed_plain": P}.get(kind, int(rng.choice([0, P, 16])))
    roles = [[counts[p], int(rng.choice([0, 0, 1, 1, 2, 3, 4])), int(rng.choice([0, 1, 2, 5, 9, 16])),
              ROLE_EXCLUSIVE if rng.random() < 0.7 else 0] for p in range(P)]
    if rng.random() < 0.15:
        roles[int(rng.integers(0, P))][1] = demand_big
    pair = rng.integers(0, 6, size=(P, Q))
    if Q and rng.random() < 0.5:
        pair[int(rng.integers(0, P))] = 0                        # all-zero pair row
    anchors: List[tuple] = []
    if Q:
        for _ in range(int(rng.integers(0, 7))):
            pool = [hubs, iso, full, None][int(rng.integers(0, 4))]
            node = int(rng.choice(pool)) if pool else int(rng.integers(0, n))
            anchors.append((node, int(rng.integers(0, Q)), int(rng.choice([0, 1, 2, 3]))))
            if rng.random() < 0.3:                               # repeated (node, q) record
                anchors.append(anchors[-1][:2] + (int(rng.integers(1, 4)),))
    consumed: List[tuple] = []
    for _ in range(int(rng.choice([0, 1, 1, 2, 4]))):
        node = int(rng.choice([a[0] for a in anchors])) if anchors and rng.random() < 0.3 else int(rng.integers(0, n))
        consumed.append((node, int(rng.choice([0, 1, 2, MAX_FREE]))))
    live = np.nonzero(topo.free > 0)[0]
    if len(live) and (kind == "consumed" or rng.random() < 0.3):
        # one node's records each fit its capacity but sum past it: a demand-0 role must lose that node; as an anchor
        # with weight toward the role it would otherwise lead the role's list
        m = int(rng.choice(live))
        consumed += [(m, int(topo.free[m])), (m, 1)]
        roles[0][1] = 0
        if Q:
            q = int(rng.integers(0, Q))
            anchors.append((m, q, 2))
            pair[0, q] = max(int(pair[0, q]), 3)
    flags = STEP_GANG if rng.random() < 0.4 else 0
    fixed = -1
    gid = int(rng.integers(0, 6))
    n_dom = len(topo.domain_owner)
    if kind == "exclusive" or (kind in ("free", "consumed") and rng.random() < 0.3):
        flags |= STEP_EXCLUSIVE
        variant = int(rng.integers(0, 6)) if kind == "exclusive" else 5
        if variant == 0:                                         # every role opted out
            for r in roles:
                r[3] = 0
        elif variant == 1:                                       # the first participating role is not role 0
            roles[0][3] = 0
            roles[1][3] = ROLE_EXCLUSIVE
        elif variant == 2:                                       # ... and is infeasible everywhere: D* = -1
            roles[0][3] = ROLE_EXCLUSIVE
            roles[0][1] = demand_big
        elif variant == 3:                                       # a fixed domain another gid owns
            owned = np.nonzero(topo.domain_owner == FOREIGN_GID)[0]
            fixed = int(rng.choice(owned)) if len(owned) else int(rng.integers(0, n_dom))
            topo.domain_owner[fixed] = FOREIGN_GID
        elif variant == 4:                                       # a domain the step's own gid owns
            d = int(rng.integers(0, n_dom))
            topo.domain_owner[d] = gid
            fixed = d if rng.random() < 0.5 else -1
        elif rng.random() < 0.4:
            fixed = int(rng.integers(0, n_dom))
    elif kind == "fixed_plain":                                  # non-exclusive: the domain is reported as -1
        fixed = int(rng.integers(0, n_dom))
    step = Step(gid=gid, roles=[tuple(r) for r in roles], pair=pair.tolist() if Q else [], anchors=anchors,
                consumed=consumed, flags=flags, fixed_domain=fixed)
    _lower_to_bound(step, limit)
    return step


def build(steps: List[Step]) -> np.ndarray:
    bb = BlobBuilder()
    for s in steps:
        bb.add(s)
    return bb.build()


def make_case(seed: int, n_nodes: int, n_steps: int) -> Case:
    """Step kinds rotate through KINDS (from an offset set by the seed), so a batch of >= 6 steps has every kind."""
    rng = np.random.default_rng(1000 + seed)
    topo, hubs, iso = topology(seed, n_nodes)
    limit = amax_limit(topo)
    steps = [_step(rng, KINDS[(s + seed) % len(KINDS)], topo, hubs, iso, limit) for s in range(n_steps)]
    return Case(topo, steps, build(steps), hubs, iso)


def hub_batch(topo, seed: int, n_small: int = 8, hub_records: int = 1, max_roles: int = MAX_STEP_ROLES) -> List[Step]:
    """Small steps (anchors on nodes of degree < 40, patch capacity far below 512) around one heavy step whose
    `hub_records` records sit on the highest-degree node; every step has 1..max_roles roles.  The heavy step's pair
    column toward the hub records is 0, so the exactness bound holds whatever the hub's weight; the weighted anchors
    elsewhere still correct its rows."""
    rng = np.random.default_rng(seed)
    deg = np.diff(topo.row_ptr)
    hub = int(np.argmax(deg))
    light = np.nonzero(deg < 40)[0]
    limit = amax_limit(topo)
    steps = []
    for s in range(n_small + 1):
        P = int(rng.integers(1, max_roles + 1))
        counts = _counts(rng, P, int(rng.integers(P, 33)))
        Q = P + 1
        roles = [(counts[p], int(rng.integers(0, 3)), int(rng.integers(0, 17)), ROLE_EXCLUSIVE if rng.random() < 0.7 else 0)
                 for p in range(P)]
        pair = rng.integers(0, 6, size=(P, Q))
        anchors = [(int(rng.choice(light)), int(rng.integers(0, Q - 1)), int(rng.integers(0, 3)))
                   for _ in range(int(rng.integers(0, 4)))]
        consumed = [(int(rng.choice(light)), int(rng.integers(0, 3))) for _ in range(int(rng.integers(0, 3)))]
        if s == n_small // 2:
            pair[:, Q - 1] = 0
            anchors += [(hub, Q - 1, 1)] * hub_records
            consumed.append((hub, 1))
        step = Step(gid=s % 5, roles=roles, pair=pair.tolist(), anchors=anchors, consumed=consumed,
                    flags=(STEP_EXCLUSIVE if s % 3 == 1 else 0) | (STEP_GANG if s % 4 == 2 else 0))
        _lower_to_bound(step, limit)
        steps.append(step)
    return steps


def exactness_edge(extra: int = 0):
    """(topo, steps) at validate_blob's bound.  tiers = 1 at N = 64: every row sums to 7 000, so the bound is
    ceil(2^24 / 15 000) = 1 119 and need·8 + Σ pair·count <= 1 118 is admitted.  Role 0 of step 0 has need 2 and
    1 102 + extra pods of its own q on one feasible node: 16 + 1 102 = 1 118 exactly, scores in [2^23, 2^24)."""
    topo = synth.make_topology(64, seed=5, tiers=1, max_free=4)
    m = int(np.nonzero(topo.free > 0)[0][0])
    steps = [Step(gid=1, roles=[(2, 1, 2, ROLE_EXCLUSIVE), (1, 0, 1, 0)], pair=[[1, 0], [0, 1]],
                  anchors=[(m, 0, 600), (m, 0, 502 + extra), (12, 1, 1)]),
             Step(gid=2, roles=[(3, 1, 1, ROLE_EXCLUSIVE)], pair=[[1]], anchors=[(40, 0, 1)], consumed=[(m, 1)])]
    return topo, steps


BULLETS = ("p8_r32", "p1_r32", "k_cap_early", "q16", "q0_consumed_only", "need_0", "need_16",
           "asym_pair_gt2", "zero_pair_row", "anchor_count_0", "anchor_count_gt1", "anchor_repeat", "anchor_full",
           "anchor_hub", "anchor_isolated",
           "cons_amount_0", "cons_amount_32767", "cons_dup_past_free", "cons_anchor", "emit_branches_one_launch",
           "fixed_non_exclusive", "fixed_foreign", "all_opt_out", "first_participant_not_0", "dstar_none",
           "self_owned", "repeat_gid",
           *[f"steps_{k}" for k in (1, 4, 5, 17, 33)], "status1_non_gang", "status2_gang",
           *[f"n_{n}" for n in (1, 3, 7, 31, 33, 130, 2049, 4097)])


def coverage(case: Case, ref=None) -> Dict[str, bool]:
    """Which limits the case reaches; `ref` = the oracle's result (status and D* bullets).

    k_cap_early: K of a role = min(replicas up to and including it, N) reaches its ceiling min(32, N) before the
    last role — with at least one replica per role that needs N < 32 (role_k clamps at N)."""
    c = dict.fromkeys(BULLETS, False)
    topo = case.topo
    n = topo.n
    deg = np.diff(topo.row_ptr)
    sizes = []
    for si, s in enumerate(case.steps):
        P, R = len(s.roles), s.n_replicas
        Q = len(s.pair[0]) if P and len(s.pair) and len(s.pair[0]) else 0
        excl = bool(s.flags & STEP_EXCLUSIVE)
        c["p8_r32"] |= P == 8 and R == 32
        c["p1_r32"] |= P == 1 and R == 32
        cum = np.cumsum([r[0] for r in s.roles])
        c["k_cap_early"] |= any(min(int(cum[p]), n) == min(KS, n) for p in range(P - 1))
        c["q16"] |= Q == 16
        c["q0_consumed_only"] |= Q == 0 and len(s.consumed) > 0
        c["need_0"] |= any(r[2] == 0 for r in s.roles)
        c["need_16"] |= any(r[2] == 16 for r in s.roles)
        if Q:
            p = np.asarray(s.pair)
            k = min(P, Q)
            c["asym_pair_gt2"] |= p.max() > 2 and bool((p[:k, :k] != p[:k, :k].T).any())
            c["zero_pair_row"] |= bool(s.anchors) and any(not p[r].any() for r in range(P))
        cnts = [a[2] for a in s.anchors]
        keys = [a[:2] for a in s.anchors]
        c["anchor_count_0"] |= 0 in cnts
        c["anchor_count_gt1"] |= any(x > 1 for x in cnts)
        c["anchor_repeat"] |= len(set(keys)) < len(keys)
        c["anchor_full"] |= any(topo.free[a[0]] == 0 for a in s.anchors)
        c["anchor_hub"] |= any(a[0] in case.hubs for a in s.anchors)
        c["anchor_isolated"] |= any(deg[a[0]] == 0 for a in s.anchors) and n > 1
        amts = [x[1] for x in s.consumed]
        c["cons_amount_0"] |= 0 in amts
        c["cons_amount_32767"] |= MAX_FREE in amts
        per: Dict[int, List[int]] = {}
        for m, a in s.consumed:
            per.setdefault(m, []).append(a)
        c["cons_dup_past_free"] |= any(len(v) > 1 and sum(v) > topo.free[m] and max(v) <= topo.free[m]
                                       for m, v in per.items())
        c["cons_anchor"] |= bool(set(per) & {a[0] for a in s.anchors})
        sizes.append(len(s.anchors) + len(s.consumed))
        c["fixed_non_exclusive"] |= not excl and s.fixed_domain >= 0
        if excl:
            own = topo.domain_owner
            part = [p for p in range(P) if s.roles[p][3] & ROLE_EXCLUSIVE]
            c["fixed_foreign"] |= s.fixed_domain >= 0 and own[s.fixed_domain] not in (-1, s.gid)
            c["all_opt_out"] |= not part
            c["first_participant_not_0"] |= s.fixed_domain < 0 and bool(part) and part[0] != 0
            c["self_owned"] |= bool((own == s.gid).any())
            if ref is not None:
                c["dstar_none"] |= s.fixed_domain < 0 and bool(part) and int(ref["domain"][si]) == -1
        if ref is not None:
            st = int(ref["status"][si])
            c["status1_non_gang"] |= st == 1 and not s.flags & STEP_GANG
            c["status2_gang"] |= st == 2
    c["emit_branches_one_launch"] = any(1 <= x <= 2 for x in sizes) and any(x > 2 for x in sizes)
    gids = [s.gid for s in case.steps]
    c["repeat_gid"] = len(set(gids)) < len(gids)
    if f"steps_{len(case.steps)}" in c:
        c[f"steps_{len(case.steps)}"] = True
    if f"n_{n}" in c:
        c[f"n_{n}"] = True
    return c
