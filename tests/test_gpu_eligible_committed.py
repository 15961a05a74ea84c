"""GPU: node eligibility in committed batches (rbgtopo_place_groups_eligible_committed[_ranked], DESIGN.md §3.20) bit for
bit against the oracle (tests/eligible_committed_oracle.py) — assign, status, domain, every pod's score and its
alternates, with the rounds of the unranked call — on generated fleets with 1, 4 and 64 classes in map and occupancy
mode; committed levels on a ctx with flags 7, including a batch whose waves have an odd step count; co-location at
levels 0 and 2 and gang-failed groups; n_alt 0, 4 and 8 and a replay across two chunks; the four reductions on one
ctx; the existing entry points unchanged by the new calls; a refresh and a re-installation of classes between calls;
every error code with nothing written and the ctx usable after it; N % 4 != 0, the room-bitmap ceiling and one above."""
import ctypes as C

import numpy as np
import pytest

import lw_commit_gen as lg
import lw_commit_levels_gen as lvg
from eligible_committed_oracle import run_eligible_committed_levels_ranked, run_eligible_committed_ranked
from eligible_oracle import ALL, full_masks
from gpu_util import new_engine
from rbg_b200 import _lib
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, STEP_GANG, Group
from rbg_b200.engine import TopoPlacer
from test_gpu_lw_limits import BITMAP_NODES, free_topo
from test_oracle_eligible import random_classes, random_masks
from test_oracle_eligible_committed import HAND_CASES, check_admitted

pytestmark = pytest.mark.gpu

EINVAL, ELIMIT = -1, -6
SENT = 0x5A5A5A5A


def bits(x):
    x = np.asarray(x)
    return x.view(np.uint32) if x.dtype == np.float32 else x


def same(got, exp, what=""):
    assert len(got) == len(exp)
    for i, (x, y) in enumerate(zip(got, exp)):
        assert np.array_equal(bits(x), bits(y)), (what, i, np.nonzero(bits(x) != bits(y))[0][:8])


def check(eng, gblob, rp, masks, exp, n_alts=(0, 4, 8)):
    """The unranked call's placement against the oracle's; for every n_alt the ranked call's placement and rounds
    equal the unranked call's and its ranking the oracle's (n_alt = 8 lists cut to n_alt)."""
    plain = eng.place_groups_eligible_committed(gblob, rp, masks)
    same(plain[:3], exp[:3], "oracle placement")
    ng = int(gblob[2])
    assert (1 if ng else 0) <= plain[3] <= max(ng, 1), plain[3]
    for F in n_alts:
        got = eng.place_groups_eligible_committed_ranked(gblob, rp, masks, F)
        same(got[:3], plain[:3], f"unranked call, n_alt {F}")
        assert got[3] == plain[3], (got[3], plain[3])
        same(got[4:], (exp[3], exp[4][:, :F], exp[5][:, :F]), f"oracle ranking, n_alt {F}")
    return plain


def fleet_engine(f, occ, **kw):
    eng = new_engine(f.topo, **kw)
    if occ:
        eng.set_exclusive_levels(f.lv[1:], f.occ)
    return eng


@pytest.mark.parametrize("seed,n,scarce", lg.SEEDS[:5])
@pytest.mark.parametrize("mode", ["map", "occupancy"])
def test_generated_fleets(seed, n, scarce, mode):
    occ = mode == "occupancy"
    f = lg.fleet(seed, n, n_groups=12, scarce=scarce, levels=occ, occupancy=occ)
    gb, rp = f.blob(), f.role_pods()
    kw = dict(level_domain=list(f.lv), owner0=lg.owner0(f)) if occ else {}
    eng = fleet_engine(f, occ)
    try:
        for k, K in enumerate((1, 4, 64)):
            cls = random_classes(n, K, seed + k)
            eng.set_node_classes(cls, K)
            masks = random_masks(gb, K, seed + k)
            exp = run_eligible_committed_ranked(f.topo, gb, rp, masks, cls, 8, **kw)
            plain = check(eng, gb, rp, masks, exp, n_alts=((0, 4, 8) if k == 1 else (4,)))
            check_admitted(gb, rp, masks, cls, plain[0])
    finally:
        eng.close()


@pytest.mark.parametrize("seed,n,scarce,kind", lvg.SEEDS[1:7])
def test_committed_levels(seed, n, scarce, kind):
    """flags 7 (RBGTOPO_CFG_LW_COMMIT_LEVELS): groups at levels 0..3, co-location at 0..3, the fleets' gang groups."""
    f = lvg.fleet(seed, n, n_groups=10, scarce=scarce, kind=kind)
    gb, rp = f.blob(), f.role_pods()
    eng = fleet_engine(f, True, lw_committed_levels=True)
    try:
        cls = random_classes(n, 6, seed)
        eng.set_node_classes(cls, 6)
        masks = random_masks(gb, 6, seed)
        exp = run_eligible_committed_levels_ranked(f.topo, gb, rp, masks, cls, 8, f.lv, f.owner(), f.nd)
        plain = check(eng, gb, rp, masks, exp, n_alts=(0, 8))
        assert lvg.violations(f.lv, f.occ, gb, rp, plain[0], plain[1]) == []
    finally:
        eng.close()


@pytest.mark.parametrize("levels", [(0, 2, 2), (2, 0, 2, 0, 2)])
def test_odd_step_waves_at_levels_with_colocation_and_gang(levels):
    """An odd number of groups, so the first wave of every round has an odd step count and the mask section of the side
    table follows an odd claim section; exclusive groups at levels 0 and 2, co-location at 0 and 2, one gang group
    that fails on its masks."""
    n = 130
    f = lvg.fleet(7, n, n_groups=len(levels), levels=levels)
    for g, grp in enumerate(f.groups):
        grp.flags |= STEP_EXCLUSIVE
        f.rp[g] = [(2, (0, 2)[(g + r) % 2]) for r in range(len(grp.roles))]
    f.groups[1].flags |= STEP_GANG
    gb, rp = f.blob(), f.role_pods()
    cls = random_classes(n, 3, 5)
    masks = random_masks(gb, 3, 5)
    r1 = len(f.groups[0].roles)
    masks[r1:r1 + len(f.groups[1].roles)] = 0   # group 1 admits no node: its gang fails
    eng = fleet_engine(f, True, lw_committed_levels=True)
    try:
        eng.set_node_classes(cls, 3)
        exp = run_eligible_committed_levels_ranked(f.topo, gb, rp, masks, cls, 8, f.lv, f.owner(), f.nd)
        assert exp[1][1] == 2 and (exp[0] >= 0).any()
        plain = check(eng, gb, rp, masks, exp)
        assert lvg.violations(f.lv, f.occ, gb, rp, plain[0], plain[1]) == []
    finally:
        eng.close()


@pytest.mark.parametrize("name", sorted(HAND_CASES))
def test_hand_built_known_answers(name):
    c = HAND_CASES[name]()
    masks = np.asarray(c["masks"], np.uint64)
    eng = new_engine(c["topo"])
    try:
        eng.set_node_classes(c["cls"], int(np.max(c["cls"])) + 1)
        exp = run_eligible_committed_ranked(c["topo"], c["blob"], c["rp"], masks, c["cls"], 8)
        check(eng, c["blob"], c["rp"], masks, exp, n_alts=(c["n_alt"],))
        got = eng.place_groups_eligible_committed_ranked(c["blob"], c["rp"], masks, c["n_alt"])
        c["expect"](got[:3] + got[4:])
    finally:
        eng.close()


def _existing(eng, gb, rp):
    return (eng.place_groups_lw_committed(gb, rp), eng.place_groups_lw_committed_ranked(gb, rp, 4),
            eng.place_groups_committed(gb), eng.place_groups_committed_ranked(gb, 4), eng.place_groups_lw(gb, rp),
            eng.place_groups_eligible(gb, rp, full_masks(gb)))


def _same_outputs(x, y):
    for a, b in zip(x, y):
        a, b = (a,) if not isinstance(a, tuple) else a, (b,) if not isinstance(b, tuple) else b
        assert len(a) == len(b)
        for u, v in zip(a, b):
            u, v = np.asarray(u), np.asarray(v)
            assert u.dtype == v.dtype and u.tobytes() == v.tobytes()


@pytest.mark.parametrize("seed,n,scarce", lg.SEEDS[1:4])
def test_reductions_and_existing_entry_points_unchanged(seed, n, scarce):
    f = lg.fleet(seed, n, n_groups=10, scarce=scarce)
    gb, rp = f.blob(), f.role_pods()
    full = full_masks(gb)
    eng = new_engine(f.topo)
    try:
        eng.set_node_classes(random_classes(n, 5, seed), 5)
        before = _existing(eng, gb, rp)
        lwc, lwcr, pc, pcr = before[:4]
        # 1. full masks: the committed leader-worker forms, rounds included; role_pods None: the committed forms
        _same_outputs([lwc], [eng.place_groups_eligible_committed(gb, rp, full)])
        _same_outputs([lwcr], [eng.place_groups_eligible_committed_ranked(gb, rp, full, 4)])
        _same_outputs([pc[:3]], [eng.place_groups_eligible_committed(gb, None, full)[:3]])
        r = eng.place_groups_eligible_committed_ranked(gb, None, full, 4)
        _same_outputs([pcr[:3] + pcr[4:]], [r[:3] + r[4:]])
        # 2. one group: the eligible call on that group
        masks = random_masks(gb, 5, seed)
        r0 = 0
        for k in range(len(f.groups)):
            one = lg.Fleet(f.topo, [f.groups[k]], [f.rp[k]], f.lv, f.occ)
            m = masks[r0:r0 + len(f.groups[k].roles)]
            r0 += len(f.groups[k].roles)
            got = eng.place_groups_eligible_committed_ranked(one.blob(), one.role_pods(), m, 4)
            assert got[3] == 1
            _same_outputs([got[:3] + got[4:]], [eng.place_groups_eligible_ranked(one.blob(), one.role_pods(), m, 4)])
        # 3. a group does not depend on the groups after it
        full_out = eng.place_groups_eligible_committed(gb, rp, masks)
        k = len(f.groups) // 2
        head = lg.Fleet(f.topo, f.groups[:k], f.rp[:k], f.lv, f.occ)
        nr = sum(len(g.roles) for g in f.groups[:k])
        a, s, d, _ = eng.place_groups_eligible_committed(head.blob(), head.role_pods(), masks[:nr])
        assert np.array_equal(a, full_out[0][:len(a)]) and np.array_equal(s, full_out[1][:k])
        assert np.array_equal(d, full_out[2][:k])
        _same_outputs(before, _existing(eng, gb, rp))   # the new calls changed no existing entry point
    finally:
        eng.close()


def test_refresh_and_reinstalled_classes_between_calls():
    f = lg.fleet(4, 130, n_groups=10, scarce=True)
    gb, rp = f.blob(), f.role_pods()
    masks = random_masks(gb, 4, 9)
    eng = new_engine(f.topo)
    try:
        for it in range(3):
            cls = random_classes(130, 4, 20 + it)
            eng.set_node_classes(cls, 4)
            exp = run_eligible_committed_ranked(f.topo, gb, rp, masks, cls, 8)
            check(eng, gb, rp, masks, exp, n_alts=(4,))
            f.topo.free = np.random.default_rng(it).integers(0, 6, 130).astype(np.int32)
            eng.update_nodes(f.topo.free, None, it + 1)
    finally:
        eng.close()


def test_a_replay_of_two_chunks_at_two_to_the_twenty_nodes():
    """2^20 nodes: a replay chunk holds 256 rows.  40 groups of one wave of 8 role rows make 320 rows: two chunks, each
    with its own mask upload, which the launch count shows (2 per chunk on top of the unranked call's)."""
    n = 1 << 20
    topo = free_topo(n, 17, max_free=2)
    topo.free[np.random.default_rng(17).random(n) > 0.01] = 0
    roles = [(0, 1, 1, ROLE_EXCLUSIVE)] * 8
    groups = [Group(gid=1 + g % 5, roles=roles, pair=[[1] * 8] * 8, anchors=[(int(g * 26_113 % n), 0, 1)],
                    flags=STEP_EXCLUSIVE if g % 2 else 0) for g in range(40)]
    gblob = lg.build(groups)
    rp = [(2 if r == 0 else 1, -1) for _ in groups for r in range(8)]
    cls = (np.arange(n) % 3).astype(np.int32)
    masks = np.asarray([(0b011, 0b110, 0b101, ALL)[r % 4] for _ in groups for r in range(8)], np.uint64)
    eng = new_engine(topo)
    try:
        eng.set_node_classes(cls, 3)
        exp = run_eligible_committed_ranked(topo, gblob, rp, masks, cls, 8)
        assert (exp[1] != 2).all() and (exp[0] >= 0).sum() > 200
        check(eng, gblob, rp, masks, exp, n_alts=(8, 1))
        eng.place_groups_eligible_committed(gblob, rp, masks)
        plain = eng.last_timing()["launches"]
        eng.place_groups_eligible_committed_ranked(gblob, rp, masks, 8)
        assert eng.last_timing()["launches"] == plain + 2 * 2, (eng.last_timing()["launches"], plain)
    finally:
        eng.close()


def raw(eng, gblob, rp, masks, n_alt, ranked):
    """The C ABI with every output filled with SENT: (rc, rounds, outputs untouched)."""
    gb = np.ascontiguousarray(gblob, np.int32)
    rpa = None if rp is None else np.ascontiguousarray(np.asarray(rp).reshape(-1), np.int32)
    mk = None if masks is None else np.ascontiguousarray(masks, np.uint64)
    outs = [np.full(4096, SENT, np.int32) for _ in range(6)]
    p = [o.ctypes.data_as(_lib.i32p) for o in outs]
    rounds = C.c_int32(SENT)
    args = [eng._h, gb.ctypes.data_as(_lib.i32p), len(gb), None if rpa is None else rpa.ctypes.data_as(_lib.i32p),
            0 if rpa is None else len(rpa), None if mk is None else mk.ctypes.data_as(_lib.u64p),
            0 if mk is None else len(mk)]
    if ranked:
        rc = eng.lib.rbgtopo_place_groups_eligible_committed_ranked(
            *args, n_alt, p[0], p[1], p[2], C.byref(rounds), C.cast(p[3], _lib.f32p), p[4], C.cast(p[5], _lib.f32p))
    else:
        rc = eng.lib.rbgtopo_place_groups_eligible_committed(*args, p[0], p[1], p[2], C.byref(rounds))
    return rc, rounds.value, all((o == SENT).all() for o in outs)


def test_error_codes_and_recovery():
    f = lg.fleet(2, 31, n_groups=6, scarce=True)
    gb, rp = f.blob(), f.role_pods()
    masks = full_masks(gb)
    eng = new_engine(f.topo)
    try:
        for ranked in (False, True):
            assert raw(eng, gb, rp, masks, 2, ranked) == (EINVAL, 0, True)             # no classes installed
        cls = random_classes(31, 3, 0)
        eng.set_node_classes(cls, 3)
        for ranked in (False, True):
            assert raw(eng, gb, rp, masks[:-1], 2, ranked) == (EINVAL, 0, True)        # one mask short
            assert raw(eng, gb, rp, None, 2, ranked) == (EINVAL, 0, True)              # no masks
            assert raw(eng, gb, rp[:-1], masks, 2, ranked) == (EINVAL, 0, True)        # role_pods short
            assert raw(eng, gb[:-1], rp, masks, 2, ranked) == (EINVAL, 0, True)        # blob short
        assert raw(eng, gb, rp, masks, 9, True) == (EINVAL, 0, True)                   # n_alt
        m = random_masks(gb, 3, 1)
        check(eng, gb, rp, m, run_eligible_committed_ranked(f.topo, gb, rp, m, cls, 8), n_alts=(2,))   # still usable
    finally:
        eng.close()
    # a group at level 1 on a ctx that places levels but not committed leader-worker levels (no flag 7)
    lvl = lg.build([Group(gid=1, roles=[(0, 1, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE, level=1)])
    lv = np.stack([f.topo.domain, np.arange(31)]).astype(np.int32)
    f.topo.domain_owner[:] = -1
    eng = new_engine(f.topo, committed_levels=True)
    try:
        eng.set_exclusive_levels(lv[1:], np.zeros((0, 3), np.int32))
        eng.set_node_classes(cls, 3)
        for ranked in (False, True):
            assert raw(eng, lvl, [(1, -1)], [ALL], 2, ranked) == (ELIMIT, 0, True)
        a, s, d, rounds = eng.place_groups_eligible_committed(gb, rp, full_masks(gb))
        assert rounds >= 1
    finally:
        eng.close()
    engs = [new_engine(f.topo, rank=r, world=2, lw_shards=True) for r in range(2)]
    try:
        for e in engs:
            e.set_node_classes(np.zeros(31, np.int32), 1)
            assert not e.places_eligible_committed
            for ranked in (False, True):
                assert raw(e, gb, rp, masks, 2, ranked) == (ELIMIT, 0, True)
            e.place_groups_lw(gb, rp)
    finally:
        for e in engs:
            e.close()


@pytest.mark.parametrize("n", [5, 130, 257])
def test_node_counts_not_a_multiple_of_four(n):
    """The slab's tail group of four: only node N - 1 (class 63) admitted for the first group's roles."""
    topo = free_topo(n, 4, max_free=2)
    topo.free[:] = 2
    gb = lg.build([Group(gid=1, roles=[(0, 1, 1, 0), (0, 1, 1, 0)], pair=[[1, 1], [1, 1]]),
                   Group(gid=2, roles=[(0, 2, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE)])
    cls = np.zeros(n, np.int32)
    cls[-1] = 63
    masks = np.asarray([1 << 63, 1 << 63, ALL], np.uint64)
    eng = new_engine(topo)
    try:
        eng.set_node_classes(cls, 64)
        exp = run_eligible_committed_ranked(topo, gb, None, masks, cls, 8)
        plain = check(eng, gb, None, masks, exp, n_alts=(2,))
        assert plain[0][0] == n - 1 and plain[0][1] == n - 1
    finally:
        eng.close()


def test_the_room_bitmap_ceiling_and_one_above():
    gb = lg.build([Group(gid=1, roles=[(0, 1, 1, 0)], pair=[[1]]), Group(gid=2, roles=[(0, 1, 1, 0)], pair=[[1]])])
    for n, code in ((BITMAP_NODES, 0), (BITMAP_NODES + 1, ELIMIT)):
        z = np.zeros(0, np.int32)
        eng = TopoPlacer(device=0)
        try:
            eng.set_topology(np.zeros(n + 1, np.int32), z, z, np.ones(n, np.int32), np.zeros(n, np.int32),
                             np.full(1, -1, np.int32))
            cls = np.zeros(n, np.int32)
            cls[-2:] = 1
            eng.set_node_classes(cls, 2)
            masks = np.asarray([0b10, 0b10], np.uint64)
            if code:
                assert raw(eng, gb, None, masks, 2, True) == (code, 0, True)
                continue
            a, s, d, rounds, sc, an, asc = eng.place_groups_eligible_committed_ranked(gb, None, masks, 2)
            assert a.tolist() == [n - 2, n - 1] and s.tolist() == [0, 0]
            assert rounds == 2   # group 1 runs again once group 0's pod is known
            assert (an == -1).all()   # both admitted nodes are full once the batch is placed
        finally:
            eng.close()
