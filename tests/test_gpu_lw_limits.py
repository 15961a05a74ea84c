"""GPU: leader-worker placement at its limits (rbgtopo_place_groups_lw / _lw_ranked / _lw_committed, DESIGN.md
§3.11-§3.13) bit for bit against the oracles (tests/lw_oracle.py, lw_alternates_oracle.py, lw_committed_oracle.py, with
the one-pass domain choice of lw_oracle.fast_domains), plus invariants read from the outputs alone: no node over free
(over the whole batch for a committed call), every replica all placed or all -1, a co-located replica inside one
level-C domain, participating pods inside the group's domain, nothing placed for a gang-failed group.

Cases: k_lw_assign's grid below the wave's step count, with co-location (the per-domain scratch bounds the grid) and
without (more steps than 8 resident 256-thread CTAs per SM); full 32-pod steps of 8 role rows competing for a few
nodes; S that does not divide 32; 16-role groups; room given back by a replica that fails part-way; ragged N with the
best node last; 32 pods of one replica stacked on one node; seven installed levels; committed claims summing past
RBGTOPO_MAX_FREE; the §3.11 rule-7 exactness bound against an enumeration of every mix of unplaced earlier pods; the
shared-memory room bitmap at exactly 1 638 400 nodes and one node past it for every call that carries it."""
import ctypes as C
import resource

import numpy as np
import pytest

import groups_gen as gg
import lw_oracle as lw
from lw_alternates_oracle import groups_of, run_lw_ranked
from lw_committed_oracle import run_lw_committed
from rbg_b200 import _lib, synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, STEP_GANG, Group, GroupsBuilder
from rbg_b200.engine import RbgTopoError, TopoPlacer, _p

pytestmark = pytest.mark.gpu

EINVAL, EINEXACT, ELIMIT = -1, -4, -6
MAX_FREE = 32767
BITMAP_NODES = 200 * 1024 * 8        # 200 KB of dynamic shared memory, one bit per node
LW_SCRATCH = 64 << 20                 # k_lw_assign's level-C domain scratch: 12 bytes per domain per CTA
SENT = 0x5A5A5A5A


def build(groups):
    gb = GroupsBuilder()
    for g in groups:
        gb.add(g)
    return gb.build()


def engine(topo, lvl=None, **kw):
    eng = TopoPlacer(device=0, **kw)
    eng.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    if lvl is not None:
        eng.set_exclusive_levels(lvl[1:], np.zeros((0, 3), np.int32))
    return eng


def free_topo(n, seed, max_free=4):
    """A snapshot without owners (co-location levels and occupancy mode need none)."""
    topo = synth.make_topology(n, seed=seed, tiers=1 if n < 8 else 2, max_free=max_free)
    topo.domain_owner[:] = -1
    return topo


def level_topo(topo, dom):
    return synth.Topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, np.asarray(dom, np.int32),
                          np.full(int(np.max(dom)) + 1, -1, np.int32))


def group_levels(gblob):
    gb = np.asarray(gblob)
    return [int(gb[8 + 12 * g + 10]) for g in range(int(gb[2]))]


def bits(x):
    return np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)


# ---- invariants read from the outputs alone

def invariants(topo, gblob, rp, lvl, a, s, d, committed=False):
    lvl = [topo.domain] if lvl is None else lvl
    free = np.asarray(topo.free, np.int64)
    batch = np.zeros(topo.n, np.int64)
    for g, X in enumerate(groups_of(gblob, rp)):
        used = np.zeros(topo.n, np.int64)
        L = group_levels(gblob)[g]
        for ri in range(X.q):
            S, Cl = X.S[ri], X.C[ri]
            base = X.pod0 + X.first_pod[ri]
            pods = a[base:base + X.pending[ri] * S].reshape(-1, S)
            assert ((pods >= 0).all(axis=1) | (pods < 0).all(axis=1)).all(), (g, ri, pods)   # all or nothing
            placed = pods[pods[:, 0] >= 0]
            if Cl >= 0 and len(placed):
                dc = np.asarray(lvl[Cl])[placed]
                assert (dc == dc[:, :1]).all(), (g, ri, placed)                           # one level-C domain
            if (X.flags & STEP_EXCLUSIVE) and (X.rflags[ri] & ROLE_EXCLUSIVE) and len(placed):
                assert (np.asarray(lvl[L])[placed] == d[g]).all(), (g, ri, d[g])          # inside domain[g]
            np.add.at(used, placed.ravel(), X.demand[ri])
        if s[g] == 2:
            assert (a[X.pod0:X.pod0 + X.n_pods] < 0).all() and used.sum() == 0, g
        assert (used <= free).all(), (g, np.nonzero(used > free)[0][:8])
        batch += used
    if committed:
        assert (batch <= free).all(), np.nonzero(batch > free)[0][:8]


# ---- the three calls against the oracles

def oracle_lw(topo, gblob, rp, lvl, n_alt):
    """run_lw_ranked per exclusive level (each level's groups against that level's partition), merged."""
    gl = group_levels(gblob)
    out = None
    with lw.fast_domains():
        for L in sorted(set(gl)):
            mine = [g for g in range(len(gl)) if gl[g] == L]
            t = topo if lvl is None else level_topo(topo, lvl[L])
            r = run_lw_ranked(t, gblob, rp, n_alt, level_domain=lvl, excl_domain=None if lvl is None else lvl[L],
                              groups=mine)
            if out is None:
                out = [np.array(x, copy=True) for x in r]
                continue
            for g in mine:
                X = groups_of(gblob, rp)[g]
                sl = slice(X.pod0, X.pod0 + X.n_pods)
                for k in (0, 3, 4, 5):
                    out[k][sl] = r[k][sl]
                out[1][g], out[2][g] = r[1][g], r[2][g]
    return out


def same(got, exp, F):
    a, s, d, sc, an, asc = got
    ea, es, ed, esc, ean, easc = exp
    assert np.array_equal(a, ea), np.nonzero(a != ea)[0][:8]
    assert np.array_equal(s, es) and np.array_equal(d, ed), (s, es, d, ed)
    assert np.array_equal(bits(sc), bits(esc)), np.nonzero(bits(sc) != bits(esc))[0][:8]
    assert np.array_equal(an, ean[:, :F]) and np.array_equal(bits(asc), bits(easc[:, :F])), \
        np.nonzero((an != ean[:, :F]).any(axis=1))[0][:8]


def run_all(eng, topo, gblob, rp, lvl=None, committed=True):
    """_lw (assign / status / domain), _lw_ranked at n_alt 0, 1, 8 (all six outputs) and, when no group is exclusive at a
    level >= 1, _lw_committed (outputs and rounds) against the oracles, each result through the invariants.
    lvl: the installed partitions, level 0 first (the ctx is then in occupancy mode without records)."""
    rp = np.asarray(rp, np.int32).reshape(-1, 2)
    exp = oracle_lw(topo, gblob, rp, lvl, 8)
    got = eng.place_groups_lw(gblob, rp)
    for x, y in zip(got, exp[:3]):
        assert np.array_equal(x, y), np.nonzero(x != y)[0][:8]
    invariants(topo, gblob, rp, lvl, *got)
    for F in (0, 1, 8):
        same(eng.place_groups_lw_ranked(gblob, rp, F), exp, F)
    if committed and max(group_levels(gblob), default=0) == 0:
        with lw.fast_domains():
            ea, es, ed = run_lw_committed(topo, gblob, rp, level_domain=lvl,
                                          owner0=None if lvl is None else np.full(topo.n, -1, np.int32))
        a, s, d, rounds = eng.place_groups_lw_committed(gblob, rp)
        assert np.array_equal(a, ea), np.nonzero(a != ea)[0][:8]
        assert np.array_equal(s, es) and np.array_equal(d, ed), (s, es, d, ed)
        ng = int(gblob[2])
        assert (1 if ng else 0) <= rounds <= max(ng, 1)
        invariants(topo, gblob, rp, lvl, a, s, d, committed=True)
    return got


def _code(fn):
    try:
        fn()
    except RbgTopoError as e:
        return e.code
    return 0


# ---- the raw ABI with sentinel-filled outputs

def raw(eng, call, gblob, rp=None, n_alt=3):
    """Calls `call` through the C ABI with every output filled with SENT; returns (rc, untouched)."""
    gb = np.ascontiguousarray(gblob, np.int32)
    ng = int(gb[2])
    if rp is not None:
        rp = np.ascontiguousarray(np.asarray(rp).reshape(-1), np.int32)
        P = TopoPlacer._lw_pods(gb, rp)
    else:
        P = int(gb[4])
    a = np.full(P + 1, SENT, np.int32)
    s, d = np.full(ng + 1, SENT, np.int32), np.full(ng + 1, SENT, np.int32)
    sc = np.full(P + 1, SENT, np.int32)
    an, asc = np.full((P + 1) * n_alt, SENT, np.int32), np.full((P + 1) * n_alt, SENT, np.int32)
    rounds = C.c_int32(0)
    f = lambda x: _p(x.view(np.float32), _lib.f32p)
    lib, h = eng.lib, eng._h
    if call == "lw":
        rc = lib.rbgtopo_place_groups_lw(h, _p(gb), len(gb), _p(rp), len(rp), _p(a), _p(s), _p(d))
    elif call == "lw_ranked":
        rc = lib.rbgtopo_place_groups_lw_ranked(h, _p(gb), len(gb), _p(rp), len(rp), n_alt, _p(a), _p(s), _p(d),
                                                f(sc), _p(an), f(asc))
    elif call == "lw_committed":
        rc = lib.rbgtopo_place_groups_lw_committed(h, _p(gb), len(gb), _p(rp), len(rp), _p(a), _p(s), _p(d),
                                                   C.byref(rounds))
    elif call == "ranked":
        rc = lib.rbgtopo_place_groups_ranked(h, _p(gb), len(gb), n_alt, _p(a), _p(s), _p(d), f(sc), _p(an), f(asc))
    else:
        assert call == "committed_ranked"
        rc = lib.rbgtopo_place_groups_committed_ranked(h, _p(gb), len(gb), n_alt, _p(a), _p(s), _p(d),
                                                       C.byref(rounds), f(sc), _p(an), f(asc))
    untouched = all((x == SENT).all() for x in (a, s, d, sc, an, asc))
    return rc, untouched


# ---- 1. k_lw_assign's grid below the wave's steps

def test_grid_below_steps_with_colocation():
    """200 000 nodes, level 1 one domain per node, level 2 racks of 16: the level-C scratch of a CTA is 12 · 200 000
    bytes, so 64 MiB hold fewer CTAs than the 72 steps of the first wave and each CTA walks several steps, reusing its
    dbest / dcap.  Most roles co-locate at 1 or 2, S in {2, 3, 4, 32}, half the nodes without room."""
    n, ng = 200_000, 72
    topo = free_topo(n, 11, max_free=3)
    rng = np.random.default_rng(11)
    topo.free = np.where(rng.random(n) < 0.5, 0, topo.free).astype(np.int32)
    lvl = [topo.domain, np.arange(n, dtype=np.int32), (np.arange(n) // 16).astype(np.int32)]
    assert ng > LW_SCRATCH // (12 * n), "the first wave must have more steps than the scratch holds CTAs"
    groups, rp = [], []
    for g in range(ng):
        S0 = 32 if g % 9 == 0 else (2, 3, 4)[g % 3]
        roles = [(0, 1, int(rng.integers(0, 3)), ROLE_EXCLUSIVE), (0, int(rng.integers(0, 3)), 1, 0)]
        groups.append(Group(gid=100 + g, roles=roles, pair=[[1, 1], [1, 1]],
                            anchors=[(int(rng.integers(0, n)), 0, 1)] if g % 2 else [],
                            flags=(STEP_EXCLUSIVE if g % 5 == 0 else 0) | (STEP_GANG if g % 4 == 3 else 0)))
        rp += [(S0, (1, 2, 1, 2, 0, -1)[g % 6]), ((2, 3, 4)[(g + 1) % 3], (2, 1, -1)[g % 3])]
    gblob = build(groups)
    eng = engine(topo, lvl)
    try:
        a, s, _ = run_all(eng, topo, gblob, rp, lvl)
        assert (a >= 0).any() and (a < 0).any() and (s == 0).any()
    finally:
        eng.close()


def test_grid_below_steps_without_colocation():
    """More steps in one wave than 8 resident 256-thread CTAs per SM (the thread ceiling, whatever the register
    count): CTAs walk several steps each.  Mixed S, anchors, 2 049 nodes."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n, ng = 2049, 8 * sms + 40
    assert ng > 8 * sms
    topo = free_topo(n, 12, max_free=6)
    rng = np.random.default_rng(12)
    groups, rp = [], []
    for g in range(ng):
        q = 1 + g % 2
        roles = [(0, int(rng.integers(1, 3)), int(rng.integers(0, 3)), 0) for _ in range(q)]
        groups.append(Group(gid=g, roles=roles, pair=[[1] * q for _ in range(q)],
                            anchors=[(int(rng.integers(0, n)), 0, int(rng.integers(1, 3)))] if g % 3 else [],
                            flags=STEP_GANG if g % 7 == 0 else 0))
        rp += [((1, 2, 3, 5)[(g + k) % 4], -1) for k in range(q)]
    gblob = build(groups)
    eng = engine(topo)
    try:
        a, s, _ = run_all(eng, topo, gblob, rp)
        assert (a >= 0).any() and 0 in s.tolist()
    finally:
        eng.close()


# ---- 2. full and odd waves

def few_nodes(n, seed, hot, free):
    topo = free_topo(n, seed, max_free=1)
    topo.free[:] = 0
    topo.free[hot] = free
    return topo


def test_full_step_of_eight_role_rows_on_a_few_nodes():
    """8 roles x S = 4 in one 32-pod step, every role competing for 6 nodes with room 6: the taken list fills up and
    room() subtracts the pods of earlier roles of the same step."""
    n = 64
    hot = [3, 9, 17, 40, 41, 63]
    topo = few_nodes(n, 21, hot, 6)
    lvl = [topo.domain, np.arange(n, dtype=np.int32), (np.arange(n) // 4).astype(np.int32)]
    roles = [(0, 1, 1 + (r % 2), 0) for r in range(8)]
    pair = [[1 if (i + j) % 3 else 0 for j in range(8)] for i in range(8)]
    for flags in (0, STEP_GANG):
        gblob = build([Group(gid=1, roles=roles, pair=pair, anchors=[(9, 0, 2)], flags=flags),
                       Group(gid=2, roles=roles[:4], pair=[p[:4] for p in pair[:4]])])
        rp = [(4, (-1, 0, 1, 2)[r % 4]) for r in range(8)] + [(4, -1)] * 4
        eng = engine(topo, lvl)
        try:
            a, s, _ = run_all(eng, topo, gblob, rp, lvl)   # 48 units of demand for 36 of room: not all of it fits
            assert s[0] == 2 if flags else ((a[:32] >= 0).any() and (a[:32] < 0).any())
        finally:
            eng.close()


def test_sizes_that_do_not_divide_32_and_a_zero_pending_role():
    n = 130
    topo = free_topo(n, 22, max_free=6)
    lvl = [topo.domain, np.arange(n, dtype=np.int32), (np.arange(n) // 16).astype(np.int32)]
    g1 = Group(gid=1, roles=[(0, 5, 1, 0), (0, 0, 1, 0), (0, 3, 0, 0), (1, 1, 1, 0)],
               pair=[[1, 1, 0, 1], [1, 1, 1, 1], [0, 1, 1, 0], [1, 0, 1, 1]], anchors=[(7, 0, 1)])
    g2 = Group(gid=2, roles=[(0, 2, 1, 0), (0, 0, 2, 0), (0, 2, 1, 0)], pair=[[1, 0, 1], [0, 1, 0], [1, 0, 1]],
               flags=STEP_GANG)
    gblob = build([g1, g2])
    eng = engine(topo, lvl)
    try:
        for rp in ([(5, 2), (7, 1), (7, -1), (31, 2), (31, 0), (1, 1), (5, -1)],
                   [(7, -1), (5, 0), (5, 2), (31, -1), (7, 2), (3, 1), (31, 0)]):
            assert any(len(w) > 1 for w in lw.pod_waves([5, 0, 3, 1], [0, 0, 0, 1], [x[0] for x in rp[:4]]))
            run_all(eng, topo, gblob, rp, lvl)
    finally:
        eng.close()


def test_sixteen_role_groups():
    n = 257
    topo = free_topo(n, 23, max_free=4)
    lvl = [topo.domain, np.arange(n, dtype=np.int32), (np.arange(n) // 16).astype(np.int32)]
    rng = np.random.default_rng(23)
    groups, rp = [], []
    for g in range(3):
        lv = np.sort(rng.integers(0, 4, size=16))
        roles = [(int(lv[i]), int(rng.integers(0, 3)), int(rng.integers(0, 2)), ROLE_EXCLUSIVE if i % 3 else 0)
                 for i in range(16)]
        pair = [[1 if i == j or rng.random() < 0.3 else 0 for j in range(16)] for i in range(16)]
        groups.append(Group(gid=g + 1, roles=roles, pair=pair, flags=(STEP_EXCLUSIVE if g != 1 else 0) |
                            (STEP_GANG if g == 2 else 0)))
        rp += [((1, 2, 3)[(i + g) % 3], (-1, 0, 1, 2)[(i * 3 + g) % 4]) for i in range(16)]
    eng = engine(topo, lvl)
    try:
        run_all(eng, topo, build(groups), rp, lvl)
    finally:
        eng.close()


def test_room_given_back_by_a_replica_that_fails_part_way():
    """Only nodes 10 and 11 have room (2 each).  Role A (S = 3, demand 2, C = -1) places two pods and fails on the
    third; role B (S = 2, demand 2) in the same step fits only in the room A gives back."""
    n = 33
    topo = few_nodes(n, 24, [10, 11], 2)
    gblob = build([Group(gid=1, roles=[(0, 1, 2, 0), (0, 1, 2, 0)], pair=[[1, 1], [1, 1]])])
    eng = engine(topo)
    try:
        a, s, _ = run_all(eng, topo, gblob, [(3, -1), (2, -1)])
        assert (a[:3] == -1).all() and sorted(a[3:].tolist()) == [10, 11] and s.tolist() == [1]
    finally:
        eng.close()


@pytest.mark.parametrize("n", [1, 31, 33, 4095, 4097])
def test_ragged_n_with_the_best_node_last(n):
    topo = free_topo(n, 25, max_free=2)
    topo.free[-1] = 64
    lvl = [topo.domain, np.arange(n, dtype=np.int32), (np.arange(n) // 16).astype(np.int32)]
    gblob = build([Group(gid=1, roles=[(0, 2, 1, 0), (0, 1, 1, 0)], pair=[[1, 1], [1, 1]], anchors=[(n - 1, 0, 6)]),
                   Group(gid=2, roles=[(0, 1, 0, 0)], pair=[[1]], anchors=[(n - 1, 0, 2)], flags=STEP_GANG)])
    eng = engine(topo, lvl)
    try:
        a, _, _ = run_all(eng, topo, gblob, [(3, 1), (4, 2), (32, 1)], lvl)
        assert (a == n - 1).any()
    finally:
        eng.close()


# ---- 3. pods stacked on one node

@pytest.mark.parametrize("demand,free", [(0, 0), (0, 3), (1, 31), (1, 32), (1, 33), (1024, MAX_FREE)])
@pytest.mark.parametrize("gang", [False, True])
def test_thirty_two_pods_stacked_on_one_node(demand, free, gang):
    """S = 32 at a level of single-node domains: the replica lands whole on one node when floor(room / demand) >= 32
    (demand 0: always), else it fails; a second role at racks of 4 spreads the same replica over a rack instead.
    Demand 1 024 with free 32 767 holds 31 pods: the per-node replica fails everywhere."""
    n = 64
    topo = free_topo(n, 26, max_free=1)
    topo.free[:] = free
    topo.free[5] = min(MAX_FREE, free + 1) if demand == 1 else free
    lvl = [topo.domain, np.arange(n, dtype=np.int32), (np.arange(n) // 4).astype(np.int32)]
    gblob = build([Group(gid=1, roles=[(0, 1, demand, 0), (0, 1, demand, 0)], pair=[[1, 1], [1, 1]],
                         anchors=[(20, 0, 1)], flags=STEP_GANG if gang else 0),
                   Group(gid=2, roles=[(0, 2, demand, 0)], pair=[[1]])])
    eng = engine(topo, lvl)
    try:
        a, s, _ = run_all(eng, topo, gblob, [(32, 1), (32, 2), (32, 1)], lvl)
        holds = demand == 0 or free // demand >= 32 or (demand == 1 and free + 1 >= 32)
        first = a[:32]
        if holds and not (gang and s[0] == 2):
            assert len(set(first.tolist())) == 1 and first[0] >= 0, first
        if demand == 1024:
            assert (first < 0).all() and (a[64:] < 0).all()
    finally:
        eng.close()


# ---- 4. seven levels

def seven_levels(n, topo):
    r = np.random.default_rng(27).permutation(n)
    return [topo.domain, np.arange(n), np.arange(n) // 2, np.arange(n) // 4, (r // 8), np.arange(n) // 16,
            np.arange(n) // 64, np.zeros(n)]


def test_seven_levels_colocation_and_exclusive_groups():
    """set_exclusive_levels with 7 levels (n_levels = RBGTOPO_MAX_EXCL_LEVELS - 1) of mixed granularity on a
    level_placement ctx: co-location on every level 0 .. 7 (7 reads the last entry of LwLevels::nd), exclusive groups at
    levels 1 .. 7, some with fixed domains; C = 8 is refused and the next call still works."""
    n = 256
    topo = free_topo(n, 27, max_free=4)
    lvl = [np.asarray(x, np.int32) for x in seven_levels(n, topo)]
    rng = np.random.default_rng(27)
    groups, rp = [], []
    for g in range(16):
        L = g % 8
        nd = int(lvl[L].max()) + 1
        excl = L > 0 or g % 2 == 0
        fixed = int(rng.integers(0, nd)) if excl and g % 3 == 0 else -1
        groups.append(Group(gid=10 + g, roles=[(0, int(rng.integers(1, 3)), 1, ROLE_EXCLUSIVE),
                                               (0, int(rng.integers(0, 3)), int(rng.integers(0, 2)), g % 2)],
                            pair=[[1, 1], [1, 1]], flags=(STEP_EXCLUSIVE if excl else 0) | (STEP_GANG if g % 5 == 4 else 0),
                            fixed_domain=fixed, level=L if excl else 0))
        rp += [((2, 3, 4)[g % 3], g % 8), ((1, 2)[g % 2], (7 - g) % 8)]
    gblob = build(groups)
    eng = engine(topo, lvl, level_placement=True)
    try:
        a, s, d = run_all(eng, topo, gblob, rp, lvl)
        assert (d >= 0).sum() >= 2 and (a >= 0).any()
        level0 = build([gr for gr in groups if gr.level == 0])
        rp0 = [x for gr, pair in zip(groups, np.asarray(rp).reshape(-1, 2, 2)) if gr.level == 0 for x in pair]
        run_all(eng, topo, level0, rp0, lvl)          # the committed call on the level-0 groups, C on every level
        bad = np.asarray(rp, np.int32).reshape(-1, 2).copy()
        bad[3, 1] = 8
        for fn in (eng.place_groups_lw, eng.place_groups_lw_committed, lambda b, r: eng.place_groups_lw_ranked(b, r, 2)):
            assert _code(lambda: fn(gblob, bad)) == EINVAL
            got = eng.place_groups_lw(gblob, rp)
            assert np.array_equal(got[0], a) and np.array_equal(got[1], s) and np.array_equal(got[2], d)
    finally:
        eng.close()


# ---- 5. committed claims past RBGTOPO_MAX_FREE

def test_committed_stale_claims_past_max_free():
    """Node 0 has free 32 767 and four groups each take 20 000 of it in round 1 (they all see an empty batch), so a
    later round stages claims summing to 40 000 and more there, clamped to RBGTOPO_MAX_FREE.  Three nodes with room
    20 000 take the groups that lose node 0; a last group of demand-0 pods anchored at node 0 follows."""
    n = 64
    topo = free_topo(n, 28, max_free=1)
    topo.free[:] = 0
    topo.free[0] = MAX_FREE
    topo.free[[30, 31, 50]] = 20_000
    big = lambda gid: Group(gid=gid, roles=[(0, 1, 20_000, 0)], pair=[[1]], anchors=[(0, 0, 4)])
    groups = [big(1), big(2), big(3), big(4),
              Group(gid=5, roles=[(0, 2, 0, 0), (0, 1, 0, 0)], pair=[[1, 1], [1, 1]], anchors=[(0, 0, 4)])]
    gblob = build(groups)
    eng = engine(topo)
    try:
        rp = [(1, -1)] * 4 + [(3, 0), (2, -1)]
        run_all(eng, topo, gblob, rp)
        a, s, _, rounds = eng.place_groups_lw_committed(gblob, rp)
        assert rounds >= 2 and (a[:4] >= 0).sum() == 4 and (a[4:] >= 0).all(), (a, s, rounds)
    finally:
        eng.close()


# ---- 6. the exactness bound of rule 7, by enumeration

def enumerated_bound(roles, pair, S, gang):
    """Per role, the largest need·F_CAP + sum_j pair·(pods of j placed before the wave) of any wave it is in, taken over
    EVERY vector u of unplaced earlier pods per role (0 .. placed_j; none for a gang group)."""
    q = len(roles)
    pend = [r[1] for r in roles]
    total = [pend[j] * S[j] for j in range(q)]
    pair = np.asarray(pair, np.int64)
    bound, placed = [0] * q, [0] * q
    for wave in lw.pod_waves(pend, [r[0] for r in roles], S):
        grids = np.meshgrid(*[np.arange(1 if gang else placed[j] + 1) for j in range(q)], indexing="ij")
        u = [x.ravel() for x in grids]
        for ri, _, _ in wave:
            need = sum(total[j] - placed[j] + u[j] for j in range(q) if pair[ri, j] > 0)
            w = sum(pair[ri, j] * (placed[j] - u[j]) for j in range(q)) + np.minimum(need, lw.NEED_CAP) * 8
            bound[ri] = max(bound[ri], int(np.max(w)))
        for ri, _, reps in wave:
            placed[ri] += reps * S[ri]
    return bound


EXACT_CASES = [   # (pair among the real roles, S, pending, gang)
    ([[1, 3], [7, 12]], (3, 1), (12, 20), False),
    ([[0, 1, 8], [3, 7, 1], [12, 0, 3]], (1, 3, 1), (10, 4, 12), True),
    ([[1, 7], [3, 0]], (32, 1), (2, 5), False),
    ([[3, 1, 12], [8, 1, 7], [1, 0, 1]], (32, 3, 1), (1, 4, 9), False),
    ([[7, 3, 1], [1, 8, 12], [0, 3, 7]], (1, 1, 32), (20, 20, 1), True),
]


def exact_group(pair, pend):
    """The real roles plus a last role with nothing pending whose pair column is 1 for every real role: its anchors
    raise every real role's anchor weight by exactly their count."""
    q = len(pend)
    roles = [(0, pend[i], 1, 0) for i in range(q)] + [(0, 0, 1, 0)]
    full = [list(pair[i]) + [1] for i in range(q)] + [[1] * (q + 1)]
    return roles, full


@pytest.mark.parametrize("pair,S,pend,gang", EXACT_CASES)
def test_exactness_bound_is_the_enumerated_worst_mix(pair, S, pend, gang):
    """At the enumerated limit all three calls refuse with RBGTOPO_EINEXACT and write nothing (raw ABI, sentinel
    outputs); one anchor less, they place and match the oracles."""
    n = 130
    topo = free_topo(n, 29, max_free=3)
    topo.free[np.random.default_rng(29).random(n) < 0.6] = 0
    roles, full = exact_group(pair, pend)
    B = enumerated_bound(roles[:-1], [r[:-1] for r in full[:-1]], list(S), gang)
    row_w = gg.wsum_max(topo) + 8000
    limit = ((1 << 24) + row_w - 1) // row_w
    c_at = limit - max(B)
    rp = [(s, -1) for s in S] + [(1, -1)]
    blob = lambda c: build([Group(gid=1, roles=roles, pair=full, anchors=[(7, len(pend), c)],
                                  flags=STEP_GANG if gang else 0)])
    eng = engine(topo)
    try:
        for call in ("lw", "lw_ranked", "lw_committed"):
            rc, untouched = raw(eng, call, blob(c_at), rp)
            assert rc == EINEXACT and untouched, (call, rc, untouched, B, c_at)
        run_all(eng, topo, blob(c_at - 1), rp)
    finally:
        eng.close()


def test_exactness_bound_attained_by_the_wave_capacity_forces():
    """One role of 40 one-pod replicas, pair weight 3, capacity for 24 pods: wave 0 (32 pods) leaves exactly 8
    unplaced, the worst mix for wave 1 (need 16, anchor weight 3 · 24), so wave 1 really stages the enumerated bound.
    One anchor under the limit it is exact and placed; at the limit the calls refuse before placing."""
    n = 130
    topo = free_topo(n, 30, max_free=1)
    topo.free[:] = 0
    topo.free[np.random.default_rng(30).choice(n, 24, replace=False)] = 1
    roles, full = exact_group([[3]], (40,))
    B = enumerated_bound(roles[:-1], [[3]], [1], False)
    assert B == [3 * 24 + 16 * 8]
    row_w = gg.wsum_max(topo) + 8000
    limit = ((1 << 24) + row_w - 1) // row_w
    blob = lambda c: build([Group(gid=1, roles=roles, pair=full, anchors=[(7, 1, c)])])
    rp = [(1, -1), (1, -1)]
    eng = engine(topo)
    try:
        for call in ("lw", "lw_ranked", "lw_committed"):
            rc, untouched = raw(eng, call, blob(limit - B[0]), rp)
            assert rc == EINEXACT and untouched, (call, rc)
        a, s, _ = run_all(eng, topo, blob(limit - B[0] - 1), rp)
        assert (a[:32] >= 0).sum() == 24 and (a[32:] < 0).all() and s.tolist() == [1]
    finally:
        eng.close()


# ---- 7. the room bitmap's ceiling

def ceiling_groups(n):
    return [Group(gid=1, roles=[(0, 2, 1, 0), (1, 1, 1, 0)], pair=[[1, 1], [1, 1]], anchors=[(n - 1, 0, 1)]),
            Group(gid=2, roles=[(0, 2, 2, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE | STEP_GANG),
            Group(gid=3, roles=[(0, 1, 0, 0)], pair=[[1]], anchors=[(123_457, 0, 2)])]


def test_room_bitmap_ceiling():
    """N = 1 638 400 fills the 200 KB room bitmap exactly: the three leader-worker calls match the oracles (level 0 cut
    into 8 domains of 204 800 nodes), place_groups_ranked equals _lw_ranked with S = 1, C = -1, and
    place_groups_committed_ranked agrees with place_groups_committed.  N = 1 638 401: every call that carries the bitmap
    returns RBGTOPO_ELIMIT with its outputs untouched, and the ctx then still places."""
    n = BITMAP_NODES
    assert (n + 31) // 32 * 4 == 200 * 1024
    topo = free_topo(n, 31, max_free=2)
    topo.domain = (np.arange(n) // (n // 8)).astype(np.int32)
    topo.domain_owner = np.full(8, -1, np.int32)
    groups = ceiling_groups(n)
    gblob = build(groups)
    eng = engine(topo)
    try:
        for rp in ([(4, 0), (2, -1), (3, 0), (32, 0)], [(2, -1), (3, 0), (1, -1), (8, -1)]):
            a, s, _ = run_all(eng, topo, gblob, rp)
            assert (a >= 0).all() and s.tolist() == [0, 0, 0]
        one = lw.role_pods_for(gblob, lambda g, r: (1, -1))
        for F in (0, 8):
            got = eng.place_groups_ranked(gblob, F)
            for x, y in zip(got, eng.place_groups_lw_ranked(gblob, one, F)):
                assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8))
            cr = eng.place_groups_committed_ranked(gblob, F)
            for x, y in zip(cr[:4], eng.place_groups_committed(gblob)):
                assert np.array_equal(x, y)
            assert (cr[4][cr[0] >= 0] != -np.inf).all()
    finally:
        eng.close()
    # one node past the bitmap: an isolated node appended to the same snapshot
    m = n + 1
    big = synth.Topology(np.append(topo.row_ptr, topo.row_ptr[-1]).astype(np.int32), topo.col_idx, topo.edge_w,
                         np.append(topo.free, 1).astype(np.int32), np.append(topo.domain, 7).astype(np.int32),
                         topo.domain_owner)
    del topo
    rp = [(4, 0), (2, -1), (3, 0), (32, 0)]
    eng = engine(big)
    try:
        for call in ("lw", "lw_ranked", "lw_committed", "ranked", "committed_ranked"):
            rc, untouched = raw(eng, call, gblob, rp if call.startswith("lw") else None)
            assert rc == ELIMIT and untouched, (call, rc, untouched)
        a, s, d = eng.place_groups(gblob)
        assert s.tolist() == [0, 0, 0] and ((a >= 0) & (a < m)).all()
        assert eng.place_groups_committed(gblob)[1].tolist() == [0, 0, 0]
    finally:
        eng.close()
    print(f"room bitmap ceiling: peak host RSS {resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1024:.0f} MiB")
