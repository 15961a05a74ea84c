"""GPU: ranked alternates of committed leader-worker batches (rbgtopo_place_groups_lw_committed_ranked, DESIGN.md
§3.15).  Every case checks all seven outputs bit for bit: assign, status, domain and rounds against
place_groups_lw_committed on the device, score, alt_node and alt_score against tests/lw_committed_alternates_oracle.py.
Cases: the lw_commit_gen fleets in map and occupancy mode with n_alt in {0, 3, 8}; exclusive groups co-located at
levels 0, 1 and 2 (k_alternates_commit_coloc); a chain of many rounds; the reductions to place_groups_committed_ranked
(commit_gen cases, occupancy cases, the bench fleet) and, for one-group batches, to place_groups_lw_ranked; 2^20 nodes
with a replay of two chunks; NULL outputs; an update_nodes between calls; and the error codes (n_alt, a level >= 1,
world = 2, one node past the room bitmap, the exactness bound), each leaving the outputs untouched and the ctx usable."""
import ctypes as C

import numpy as np
import pytest

import commit_gen as cg
import groups_gen as gg
import lw_commit_gen as lg
import lw_oracle as lw
from gpu_util import new_engine
from lw_committed_alternates_oracle import run_lw_committed_ranked
from rbg_b200 import _lib, synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, Group
from rbg_b200.engine import RbgTopoError, TopoPlacer
from test_gpu_lw_limits import BITMAP_NODES, enumerated_bound, exact_group, free_topo

pytestmark = pytest.mark.gpu

EINVAL, EINEXACT, ELIMIT = -1, -4, -6
SENT = 0x5A5A5A5A


def bits(x):
    x = np.asarray(x)
    return x.view(np.uint32) if x.dtype == np.float32 else x


def same(got, exp, what=""):
    for i, (x, y) in enumerate(zip(got, exp)):
        assert np.array_equal(bits(x), bits(y)), (what, i, np.nonzero(bits(x) != bits(y))[0][:8])


def check(eng, topo, gblob, rp, n_alts=(0, 3, 8), exp=None, **oracle_kw):
    """All seven outputs for every n_alt: placement and rounds against place_groups_lw_committed, the ranking against
    the oracle (alternates for a smaller n_alt are the prefix of the oracle's n_alt = 8 lists)."""
    plain = eng.place_groups_lw_committed(gblob, rp)
    if exp is None:
        exp = run_lw_committed_ranked(topo, gblob, rp, 8, **oracle_kw)
    same(plain[:3], exp[:3], "oracle placement")
    got = None
    for F in n_alts:
        got = eng.place_groups_lw_committed_ranked(gblob, rp, F)
        same(got[:3], plain[:3], f"place_groups_lw_committed, n_alt {F}")
        assert got[3] == plain[3], (got[3], plain[3])
        same(got[4:], (exp[3], exp[4][:, :F], exp[5][:, :F]), f"oracle ranking, n_alt {F}")
    return got


def fleet_engine(f: lg.Fleet, occ: bool):
    eng = new_engine(f.topo)
    if occ:
        eng.set_exclusive_levels(f.lv[1:], f.occ)
    return eng


def fleet_kw(f: lg.Fleet, occ: bool):
    return dict(level_domain=list(f.lv), owner0=lg.owner0(f)) if occ else {}


@pytest.mark.parametrize("seed,n,scarce", lg.SEEDS)
@pytest.mark.parametrize("mode", ["map", "occupancy"])
def test_seeded_fleets(seed, n, scarce, mode):
    occ = mode == "occupancy"
    f = lg.fleet(seed, n, n_groups=14, scarce=scarce, levels=occ, occupancy=occ)
    eng = fleet_engine(f, occ)
    try:
        got = check(eng, f.topo, f.blob(), f.role_pods(), **fleet_kw(f, occ))
        assert (got[5] >= 0).any() or n < 16
    finally:
        eng.close()


@pytest.mark.parametrize("level", [0, 1, 2])
def test_exclusive_groups_colocated_at_every_level(level):
    """Every group exclusive, every role co-located at `level`: the jobs carry both the owner test and the
    co-location domain (k_alternates_commit_coloc); level 1 has single-node domains, so no pod has an alternate."""
    f = lg.fleet(7, 257, n_groups=12, levels=True, occupancy=True)
    for g in f.groups:
        g.flags |= STEP_EXCLUSIVE
    f.rp = [[(S, level) for S, _ in rp] for rp in f.rp]
    eng = fleet_engine(f, True)
    try:
        got = check(eng, f.topo, f.blob(), f.role_pods(), **fleet_kw(f, True))
        placed = got[0] >= 0
        assert placed.any()
        if level == 1:
            assert (got[5] == -1).all()
        else:
            assert (got[5][placed] >= 0).any()
            lv = f.lv[level]
            for p in np.nonzero(placed)[0]:
                alt = got[5][p][got[5][p] >= 0]
                assert (lv[alt] == lv[got[0][p]]).all()
    finally:
        eng.close()


def test_a_chain_of_many_rounds_ranks_each_groups_final_run():
    case = cg.chain(24, 48, 3)
    rp = lw.role_pods_for(case.blob, lambda g, r: (2, -1))
    eng = new_engine(case.topo)
    try:
        got = check(eng, case.topo, case.blob, rp)
        assert got[3] > 2
    finally:
        eng.close()


def _without_rounds(x):
    return x[:3] + x[4:]


@pytest.mark.parametrize("k", range(len(cg.cases())))
def test_one_pod_per_replica_is_place_groups_committed_ranked(k):
    case = cg.cases()[k]
    rp = lw.role_pods_for(case.blob, lambda g, r: (1, -1))
    eng = new_engine(case.topo)
    try:
        for F in (0, 8):
            same(_without_rounds(eng.place_groups_lw_committed_ranked(case.blob, rp, F)),
                 _without_rounds(eng.place_groups_committed_ranked(case.blob, F)), case.name)
    finally:
        eng.close()


def test_one_pod_per_replica_in_occupancy_mode_and_on_the_bench_fleet():
    for case, lv, occ, _ in cg.occupancy_cases():
        eng = new_engine(case.topo)
        try:
            eng.set_exclusive_levels(lv[1:], occ)
            rp = lw.role_pods_for(case.blob, lambda g, r: (1, -1))
            same(_without_rounds(eng.place_groups_lw_committed_ranked(case.blob, rp, 8)),
                 _without_rounds(eng.place_groups_committed_ranked(case.blob, 8)), case.name)
        finally:
            eng.close()
    import bench
    from rbg_b200.plugin import B200TopoPodGroupManager
    topo = synth.make_topology(4096, seed=3)
    eng = new_engine(topo)
    try:
        gblob, _ = B200TopoPodGroupManager(eng).groups_blob(bench.to_plugin(bench.fleet_spec("mooncake", 64, 4096, 3)))
        rp = lw.role_pods_for(gblob, lambda g, r: (1, -1))
        for F in (3, 8):
            same(_without_rounds(eng.place_groups_lw_committed_ranked(gblob, rp, F)),
                 _without_rounds(eng.place_groups_committed_ranked(gblob, F)), "bench fleet")
    finally:
        eng.close()


@pytest.mark.parametrize("seed,n,scarce", lg.SEEDS[:4])
def test_one_group_batches_are_place_groups_lw_ranked(seed, n, scarce):
    f = lg.fleet(seed, n, scarce=scarce)
    eng = new_engine(f.topo)
    try:
        for k in range(len(f.groups)):
            one = lg.Fleet(f.topo, [f.groups[k]], [f.rp[k]], f.lv, f.occ)
            for F in (0, 8):
                got = eng.place_groups_lw_committed_ranked(one.blob(), one.role_pods(), F)
                same(_without_rounds(got), eng.place_groups_lw_ranked(one.blob(), one.role_pods(), F), f"group {k}")
                assert got[3] == 1
    finally:
        eng.close()


def test_a_replay_of_two_chunks_at_two_to_the_twenty_nodes():
    """2^20 nodes: slab_stride 2^20, so a replay chunk holds 256 rows.  40 groups of one wave of 8 role rows each
    make 320 rows: two chunks, which the launch count shows (2 per chunk on top of place_groups_lw_committed's)."""
    n = 1 << 20
    topo = free_topo(n, 17, max_free=2)
    topo.free[np.random.default_rng(17).random(n) > 0.01] = 0
    roles = [(0, 1, 1, ROLE_EXCLUSIVE)] * 8
    groups = [Group(gid=1 + g % 5, roles=roles, pair=[[1] * 8] * 8, anchors=[(int(g * 26_113 % n), 0, 1)],
                    flags=STEP_EXCLUSIVE if g % 2 else 0) for g in range(40)]
    gblob = lg.build(groups)
    rp = [(2 if r == 0 else 1, -1) for _ in groups for r in range(8)]
    eng = new_engine(topo)
    try:
        exp = run_lw_committed_ranked(topo, gblob, rp, 8)
        assert (exp[1] != 2).all() and all((exp[0][9 * g:9 * g + 9] >= 0).any() for g in range(40))
        check(eng, topo, gblob, rp, n_alts=(8, 1), exp=exp)
        eng.place_groups_lw_committed(gblob, rp)
        plain = eng.last_timing()["launches"]
        eng.place_groups_lw_committed_ranked(gblob, rp, 8)
        assert eng.last_timing()["launches"] == plain + 2 * 2, (eng.last_timing()["launches"], plain)
    finally:
        eng.close()


def raw(eng, gblob, rp, n_alt, null_status=False, null_alt=False):
    """The C ABI with every output filled with SENT: (rc, outputs)."""
    gb = np.ascontiguousarray(gblob, np.int32)
    rp = np.ascontiguousarray(np.asarray(rp).reshape(-1), np.int32)
    ng, P = int(gb[2]), TopoPlacer._lw_pods(gb, rp)
    F = max(n_alt, 0)
    out = dict(a=np.full(P + 1, SENT, np.int32), s=np.full(ng + 1, SENT, np.int32), d=np.full(ng + 1, SENT, np.int32),
               sc=np.full(P + 1, SENT, np.int32), an=np.full((P + 1) * F + 1, SENT, np.int32),
               asc=np.full((P + 1) * F + 1, SENT, np.int32))
    rounds = C.c_int32(SENT)
    p = lambda k, t=_lib.i32p: out[k].ctypes.data_as(t)
    rc = eng.lib.rbgtopo_place_groups_lw_committed_ranked(
        eng._h, gb.ctypes.data_as(_lib.i32p), len(gb), rp.ctypes.data_as(_lib.i32p), len(rp), n_alt, p("a"),
        None if null_status else p("s"), None if null_status else p("d"), None if null_status else C.byref(rounds),
        p("sc", _lib.f32p), None if null_alt else p("an"), None if null_alt else p("asc", _lib.f32p))
    out["rounds"] = rounds.value
    return rc, out


def untouched(out):
    return all((v == SENT).all() for k, v in out.items() if k != "rounds")


def test_null_outputs_and_update_nodes_between_calls():
    f = lg.fleet(21, 257, n_groups=10, scarce=True)
    gb, rp = f.blob(), f.role_pods()
    eng = new_engine(f.topo)
    try:
        ref = check(eng, f.topo, gb, rp, n_alts=(8,))
        P = len(ref[0])
        rc, out = raw(eng, gb, rp, 8, null_status=True)
        assert rc == 0
        same((out["a"][:P], out["sc"][:P].view(np.float32), out["an"][:P * 8].reshape(P, 8),
              out["asc"][:P * 8].view(np.float32).reshape(P, 8)), (ref[0], ref[4], ref[5], ref[6]), "NULL status")
        rc, out = raw(eng, gb, rp, 0, null_status=True, null_alt=True)
        assert rc == 0
        same((out["a"][:P], out["sc"][:P].view(np.float32)), (ref[0], ref[4]), "n_alt 0, NULL alternates")
        rng = np.random.default_rng(0)
        f.topo.free = rng.integers(0, 4, f.topo.n).astype(np.int32)
        eng.update_nodes(f.topo.free)
        check(eng, f.topo, gb, rp, n_alts=(3,))
        nodes = np.arange(0, f.topo.n, 7, dtype=np.int32)
        f.topo.free[nodes] = 6
        eng.update_nodes_delta(nodes, f.topo.free[nodes])
        check(eng, f.topo, gb, rp, n_alts=(8,))
    finally:
        eng.close()


def test_error_codes_write_nothing_and_leave_the_ctx_usable():
    f = lg.fleet(31, 64, n_groups=4)
    gb, rp = f.blob(), f.role_pods()
    lv = np.stack([f.topo.domain, np.arange(64) // 8]).astype(np.int32)
    lvl = Group(gid=3, roles=[(0, 1, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE, level=1)
    lvl_blob = lg.build(f.groups + [lvl])
    lvl_rp = np.concatenate([rp, [[2, -1]]])
    eng, flagged = new_engine(f.topo), new_engine(f.topo, committed_levels=True)
    try:
        for F in (9, -1):
            rc, out = raw(eng, gb, rp, F)
            assert rc == EINVAL and untouched(out) and out["rounds"] == 0, (F, rc)
        rc, out = raw(eng, gb, rp, 4, null_alt=True)
        assert rc == EINVAL and untouched(out)
        for e in (eng, flagged):
            e.set_exclusive_levels(lv[1:], np.zeros((0, 3), np.int32))
            rc, out = raw(e, lvl_blob, lvl_rp, 4)
            assert rc == ELIMIT and untouched(out) and out["rounds"] == 0, rc
            kw = dict(level_domain=list(lv), owner0=np.full(64, -1, np.int32))
            check(e, f.topo, gb, rp, n_alts=(4,), **kw)
    finally:
        eng.close()
        flagged.close()
    engs = [new_engine(f.topo, rank=r, world=2) for r in range(2)]
    try:
        for e in engs:
            rc, out = raw(e, gb, rp, 4)
            assert rc == ELIMIT and untouched(out)
            e.place_groups(gb)
    finally:
        for e in engs:
            e.close()


def test_one_node_past_the_room_bitmap():
    m = BITMAP_NODES + 1
    topo = free_topo(m, 31, max_free=2)
    groups = [Group(gid=1, roles=[(0, 2, 1, 0), (1, 1, 1, 0)], pair=[[1, 1], [1, 1]], anchors=[(m - 1, 0, 1)])]
    gb = lg.build(groups)
    rp = [(4, 0), (2, -1)]
    eng = new_engine(topo)
    try:
        rc, out = raw(eng, gb, rp, 8)
        assert rc == ELIMIT and untouched(out) and out["rounds"] == 0, rc
        with pytest.raises(RbgTopoError) as ex:
            eng.place_groups_lw_committed(gb, rp)
        assert ex.value.code == ELIMIT
        a, s, _ = eng.place_groups(gb)
        assert s.tolist() == [0] and ((a >= 0) & (a < m)).all()
    finally:
        eng.close()


def test_the_exactness_bound_is_place_groups_lw_committeds():
    """At the enumerated limit of §3.11 rule 7 both calls refuse with RBGTOPO_EINEXACT and the ranked one writes
    nothing; one anchor less, both place and the ranked call matches the oracle."""
    pair, S, pend = [[1, 3], [7, 12]], (3, 1), (12, 20)
    n = 130
    topo = free_topo(n, 29, max_free=3)
    topo.free[np.random.default_rng(29).random(n) < 0.6] = 0
    roles, full = exact_group(pair, pend)
    B = enumerated_bound(roles[:-1], [r[:-1] for r in full[:-1]], list(S), False)
    row_w = gg.wsum_max(topo) + 8000
    c_at = ((1 << 24) + row_w - 1) // row_w - max(B)
    rp = [(s, -1) for s in S] + [(1, -1)]
    blob = lambda c: lg.build([Group(gid=1, roles=roles, pair=full, anchors=[(7, len(pend), c)])])
    eng = new_engine(topo)
    try:
        with pytest.raises(RbgTopoError) as ex:
            eng.place_groups_lw_committed(blob(c_at), rp)
        assert ex.value.code == EINEXACT
        rc, out = raw(eng, blob(c_at), rp, 8)
        assert rc == EINEXACT and untouched(out) and out["rounds"] == 0, rc
        check(eng, topo, blob(c_at - 1), rp, n_alts=(8,))
    finally:
        eng.close()
