"""GPU: committed batches (DESIGN.md §3.8) at the limits of their round machinery, bit for bit against the committed
oracle (tests/committed_oracle.py) — assign, status and domain of every group: the generated batches of
tests/commit_gen.py with their known round counts (full chains, claims that move or vanish, domain claims, a hub's
long claim list, claims read through the table, N = 1 .. 4097), world 2 and 4 contexts, occupancy mode (§3.9) with
records at every level, snapshot refreshes that run while a committed call is in its rounds, and a group's table on both
sides of the shared-memory ceiling."""
import threading
import time

import numpy as np
import pytest

import commit_gen as cg
import groups_gen as gg
import levels_oracle as lo
from committed_oracle import result_arrays, run_fleet_committed
from gpu_util import new_engine
from oracle import wave_loop
from rbg_b200 import synth

pytestmark = pytest.mark.gpu

CASES = cg.cases()
KEYS = [f"example.com/level-{L}" for L in range(8)]


def pending_groups(gblob):
    return sum(1 for g in range(int(gblob[2])) if int(gblob[8 + 12 * g + 9]) > 0)


def expected(topo, gblob, owner0=None):
    return result_arrays(run_fleet_committed(topo, wave_loop.groups_from_blob(gblob), owner0=owner0, fast=True))


def same(got, exp):
    return all(np.array_equal(np.asarray(x), np.asarray(y)) for x, y in zip(got[:3], exp))


def check(eng, topo, gblob, owner0=None):
    got = eng.place_groups_committed(gblob)
    ea, es, ed = expected(topo, gblob, owner0)
    a, s, d, rounds = got
    assert np.array_equal(a, ea), np.nonzero(a != ea)[0][:8]
    assert np.array_equal(s, es), (np.nonzero(s != es)[0][:8], s[:16], es[:16])
    assert np.array_equal(d, ed), (np.nonzero(d != ed)[0][:8], d[:16], ed[:16])
    n0 = pending_groups(gblob)
    assert (rounds == 0) if n0 == 0 else (1 <= rounds <= n0), (rounds, n0)
    return got


@pytest.mark.parametrize("i", range(len(CASES)), ids=[c.name for c in CASES])
def test_generated_batches_match_the_oracle(i):
    case = CASES[i]
    eng = new_engine(case.topo)
    try:
        a, s, d, rounds = check(eng, case.topo, case.blob)
        if case.rounds is not None:
            assert rounds == case.rounds, (rounds, case.rounds)
        if "chain" in case.tags:     # every chain group gets a node, the one without idle groups on the host's bound
            assert (s == 0).all() and (a >= 0).all()
            assert ("chain_n0_eq_ng" not in case.tags) or rounds == int(case.blob[2])
    finally:
        eng.close()


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("n", [130, 4097])
def test_world_contexts_equal_world_1_and_the_oracle(world, n):
    cs = [cg.scarce(60 + n, n, n_groups=24), cg.domains(61 + n, n), cg.chain(24, n, 62)]
    for case in cs:
        e1 = new_engine(case.topo)
        try:
            ref = check(e1, case.topo, case.blob)
        finally:
            e1.close()
        engs = [new_engine(case.topo, rank=r, world=world) for r in range(world)]
        try:
            for e in engs:
                r = e.place_groups_committed(case.blob)
                assert same(r, ref[:3]) and r[3] == ref[3], (case.name, e)
        finally:
            for e in engs:
                e.close()


def check_records(lv, occ, gblob, assign, status):
    """The GPU's own placements of exclusive groups' participating roles keep the records' anti-affinity terms."""
    groups = wave_loop.groups_from_blob(gblob)
    off = 0
    for g in groups:
        s = wave_loop.GroupState(g)
        for ri in s.order:
            r = g.roles[ri]
            for c in range(s.pending[ri]):
                node = int(assign[off])
                off += 1
                if g.exclusive and r.exclusive and node >= 0:
                    assert not lo.violates(lv, KEYS[:len(lv)], occ, g.gid, 0, node), (g.name, r.name, node)


def test_occupancy_known_answer():
    """A claim never unblocks a node the records block: the second gid-7 group gets no node (DESIGN.md §3.9)."""
    topo, lv, occ, _, gblob = cg.known_occupancy()
    eng = new_engine(topo)
    try:
        eng.set_exclusive_levels(lv[1:], occ)
        owner0 = lo.derive_level_owner(lv, occ)[0]
        a, s, d, _ = check(eng, topo, gblob, owner0)
        assert a.tolist() == [0, -1] and d.tolist() == [0, -1]
        check_records(lv, occ, gblob, a, s)
    finally:
        eng.close()


@pytest.mark.parametrize("i", range(len(cg.occupancy_cases())))
def test_occupancy_batches_match_the_oracle_and_keep_the_records(i):
    case, lv, occ, owner0 = cg.occupancy_cases()[i]
    eng = new_engine(case.topo)
    try:
        eng.set_exclusive_levels(lv[1:], occ)
        assert np.array_equal(eng.read_snapshot("level_owner")[0], owner0)
        a, s, d, _ = check(eng, case.topo, case.blob, owner0)
        check_records(lv, occ, case.blob, a, s)
    finally:
        eng.close()
    if i == 1:
        engs = [new_engine(case.topo, rank=r, world=2) for r in range(2)]
        try:
            for e in engs:
                e.set_exclusive_levels(lv[1:], occ)
                r = e.place_groups_committed(case.blob)
                assert same(r, (a, s, d))
        finally:
            for e in engs:
                e.close()


def _refreshed(case, kind):
    """(the refresh as a call on an engine, the snapshot it installs as (topo, owner0))."""
    topo = case.topo
    if kind == "levels":
        lv = lo.random_levels(np.random.default_rng(5), topo.n, topo.domain, 3, [True, False, True])
        occ = lo.random_occ(np.random.default_rng(6), topo.n, 3, [7, 8], topo.n // 4)
        return (lambda e: e.set_exclusive_levels(lv[1:], occ)), topo, lo.derive_level_owner(lv, occ)[0]
    new = synth.Topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free.copy(), topo.domain, topo.domain_owner)
    nodes = np.arange(0, topo.n, 3, dtype=np.int32)
    new.free[nodes] = 0
    if kind == "free":
        return (lambda e: e.update_nodes(free=new.free)), new, None
    return (lambda e: e.update_nodes_delta(nodes, np.zeros(len(nodes), np.int32))), new, None


@pytest.mark.parametrize("kind", ["free", "delta", "levels"])
def test_a_refresh_during_a_call_lands_between_calls(kind, record_property):
    """A chain of 300 groups (300 rounds) in one thread, one refresh in another, issued 2 ms into the call: the call's
    result is the oracle's on exactly one of the two snapshots, and the ctx places on the new one afterwards.  Which
    snapshot the call saw, the call's duration and when the refresh returned are recorded (junit properties): a call
    that outlasts the 2 ms and still saw the old snapshot held the refresh back until its last round."""
    case = cg.chain(300, 320, 70)
    if kind == "levels":   # one gid: the chain's exclusive groups share domains, the records block some nodes
        for g in case.groups:
            g.gid, g.flags = 7, cg.STEP_EXCLUSIVE
        case.blob = cg.build(case.groups)
    refresh, new_topo, new_owner0 = _refreshed(case, kind)
    old = expected(case.topo, case.blob)
    new = expected(new_topo, case.blob, new_owner0)
    assert not all(np.array_equal(x, y) for x, y in zip(old, new))
    eng = new_engine(case.topo)
    try:
        out = {}
        started = threading.Event()

        def call():
            started.set()
            t0 = time.perf_counter()
            out["r"] = eng.place_groups_committed(case.blob)
            out["call"] = (t0, time.perf_counter())
        t = threading.Thread(target=call)
        t.start()
        started.wait()
        time.sleep(0.002)
        r0 = time.perf_counter()
        refresh(eng)
        r1 = time.perf_counter()
        t.join()
        r = out["r"]
        assert same(r, old) != same(r, new), "a result mixed of two snapshots"
        c0, c1 = out["call"]
        seen = "old" if same(r, old) else "new"
        record_property("snapshot_seen", seen)
        record_property("call_ms", round(1e3 * (c1 - c0), 3))
        record_property("refresh_issued_ms", round(1e3 * (r0 - c0), 3))
        record_property("refresh_returned_ms", round(1e3 * (r1 - c0), 3))
        record_property("rounds", int(r[3]))
        again = eng.place_groups_committed(case.blob)
        assert same(again, new)
    finally:
        eng.close()


def test_tables_on_both_sides_of_the_shared_memory_ceiling():
    """A 16-role group whose table of patched nodes is the largest that fits shared memory is placed like the oracle;
    one more scheduled pod's neighbourhood takes its table (rbgtopo_place_describe geom[4]) past the ceiling, and the
    call returns RBGTOPO_ELIMIT before anything runs on the device."""
    from test_gpu_groups_limits import _one_role_groups, _wide_group
    from test_place_describe import describe
    from rbg_b200.engine import RbgTopoError
    n = 4097
    rng = np.random.default_rng(121)
    topo = synth.make_topology(n, seed=3, tiers=4, max_free=4)
    wide = _wide_group(rng, 16, 5, n)
    p = np.asarray(wide.pair)
    p[:, 15] = 0
    wide.pair = p.tolist()
    nodes = rng.permutation(n)
    others = _one_role_groups(rng, 20, 10, n)

    def batch(k):
        wide.anchors = [(int(x), 15, 1) for x in nodes[:k]]
        return cg.build(others[:3] + [wide] + others[3:])
    eng = new_engine(topo)
    try:
        def fits(k):
            try:
                eng.place_groups_committed(batch(k))
                return True
            except RbgTopoError as e:
                assert e.code == -6, e
                return False
        lo_k, hi_k = 0, 1
        while fits(hi_k):
            lo_k, hi_k = hi_k, 2 * hi_k
        while hi_k - lo_k > 1:
            mid = (lo_k + hi_k) // 2
            lo_k, hi_k = (mid, hi_k) if fits(mid) else (lo_k, mid)
        degp1 = (np.diff(topo.row_ptr) + 1).astype(np.int32)
        (rc0, g0, _), (rc1, g1, _) = (describe(batch(k), topo, degp1, gg.wsum_max(topo)) for k in (lo_k, lo_k + 1))
        assert rc0 == rc1 == 0 and g1[4] > g0[4] and lo_k > 0, (lo_k, g0, g1)
        with pytest.raises(RbgTopoError) as e:
            eng.place_groups_committed(batch(lo_k + 1))
        assert e.value.code == -6 and "shared memory" in str(e.value)
        check(eng, topo, batch(lo_k))
    finally:
        eng.close()
