"""GPU: node eligibility (rbgtopo_set_node_classes, rbgtopo_place_groups_eligible[_ranked], DESIGN.md §3.19) bit for
bit against the oracle (tests/eligible_oracle.py) — assign, status, domain, every pod's score and its alternates — on
generated fleets with 1 to 64 classes, the mooncake and fleet8 shapes, exclusive groups at levels 0 and 2 with
co-location, scarce capacity and n_alt 0 to 8; with full masks, the four forms it reduces to on the same ctx; the
existing entry points unchanged by installed classes; slab edges (N = 1, N % 4 != 0, a one-node chunk tail, class 63,
only node N - 1 admitted, N = 2^20 + 1, the room-bitmap ceiling); ordering behind an in-flight call on a caller
stream; set_topology dropping the classes; every error code followed by a call that works."""
import numpy as np
import pytest

import groups_gen as gg
import lw_oracle as lw
from eligible_oracle import ALL, full_masks, run_eligible, run_eligible_ranked
from rbg_b200 import synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, STEP_GANG, Group
from rbg_b200.engine import TopoPlacer
from test_gpu_lw import _code, build, cycle_pods, level_setup, level_topo
from test_gpu_lw_alternates import same
from test_oracle_eligible import HAND_CASES, random_classes, random_masks

pytestmark = pytest.mark.gpu


def engine(topo, **kw):
    eng = TopoPlacer(device=0, **kw)
    eng.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    return eng


def check(eng, topo, gblob, rp, masks, cls, n_alt, **kw):
    """The ranked call against the oracle, its assign / status / domain equal to the unranked call's."""
    got = eng.place_groups_eligible_ranked(gblob, rp, masks, n_alt)
    for x, y in zip(got[:3], eng.place_groups_eligible(gblob, rp, masks)):
        assert np.array_equal(x, y)
    same(got, run_eligible_ranked(topo, gblob, rp, masks, cls, n_alt, **kw))
    return got


@pytest.mark.parametrize("seed,n,scarce,excl", gg.CASES)
def test_generated_fleets(seed, n, scarce, excl):
    case = gg.make_case(seed, n, scarce=scarce, exclusive=excl)
    eng = engine(case.topo)
    try:
        for k, (K, F) in enumerate(((1, 0), (2, 1), (7, 3), (64, 8))):
            cls = random_classes(n, K, seed + k)
            eng.set_node_classes(cls, K)
            masks = random_masks(case.blob, K, seed + k)
            rp = (cycle_pods(case.blob), None, cycle_pods(case.blob, S=(4, 2), C=(0,)), None)[k]
            check(eng, case.topo, case.blob, rp, masks, cls, F)
    finally:
        eng.close()


@pytest.mark.parametrize("shape,seed", [("mooncake", 0), ("fleet8", 1)])
def test_fleet_shapes(shape, seed):
    import bench
    from rbg_b200.plugin import B200TopoPodGroupManager
    n = 2049
    topo = synth.make_topology(n, seed=seed)
    eng = engine(topo)
    try:
        gblob, runs = B200TopoPodGroupManager(eng).groups_blob(bench.to_plugin(bench.fleet_spec(shape, 24, n, seed)))
        cls = (np.arange(n) % 3 == 0).astype(np.int32)   # class 1: a third of the nodes, the GPU pool
        eng.set_node_classes(cls, 2)
        rp, masks = [], []
        for i, g in enumerate(runs):
            for ri in g.order:
                name = g.rbg.roles[ri].name
                gpu = "prefill" in name or "decode" in name
                rp.append((2 if gpu and i % 2 else 1, (0, -1)[i % 3 == 2]))
                masks.append(0b10 if gpu else 0b01)   # CPU roles do not tolerate the GPU pool
        got = check(eng, topo, gblob, rp, np.asarray(masks, np.uint64), cls, 3)
        assert (got[0] >= 0).any() and (got[4] >= 0).any()
    finally:
        eng.close()


@pytest.mark.parametrize("seed,n", [(1, 33), (3, 2049)])
def test_exclusive_levels_and_colocation(seed, n):
    """Exclusive groups at levels 0 and 2 on a LEVEL_PLACEMENT ctx (occupancy mode), co-location at 0, 1 and 2."""
    topo, lv = level_setup(n, seed)
    rng = np.random.default_rng(seed)
    groups, levels = [], []
    for g in range(8):
        L = (0, 2)[g % 2]
        excl = g % 3 != 1
        roles = [(0, int(rng.integers(1, 4)), int(rng.integers(0, 3)), ROLE_EXCLUSIVE),
                 (1, int(rng.integers(1, 3)), 1, ROLE_EXCLUSIVE if g % 2 else 0)]
        groups.append(Group(gid=10 + g, roles=roles, pair=[[1, 1], [1, 1]], anchors=[(int(rng.integers(0, n)), 0, 1)],
                            flags=STEP_EXCLUSIVE if excl else 0, level=L))
        levels.append(L)
    cls = random_classes(n, 4, seed)
    eng = engine(topo, level_placement=True)
    try:
        eng.set_exclusive_levels(lv[1:], np.zeros((0, 3), np.int32))
        eng.set_node_classes(cls, 4)
        for g, L in enumerate(levels):   # each group against the oracle at its own level
            gblob = build([groups[g]])
            rp = [(2, (0, 1, 2)[g % 3]), (1, -1)]
            masks = random_masks(gblob, 4, seed + g)
            check(eng, level_topo(topo, lv[L]), gblob, rp, masks, cls, g % 5, level_domain=lv, excl_domain=lv[L])
    finally:
        eng.close()


@pytest.mark.parametrize("name", sorted(HAND_CASES))
def test_hand_built_known_answers(name):
    c = HAND_CASES[name]()
    eng = engine(c["topo"])
    try:
        eng.set_node_classes(c["cls"], int(np.max(c["cls"])) + 1)
        got = check(eng, c["topo"], c["blob"], c["rp"], np.asarray(c["masks"], np.uint64), c["cls"], c["n_alt"])
        c["expect"](got)
    finally:
        eng.close()


def _outputs(eng, case, rp):
    return (eng.place_groups(case.blob), eng.place_groups_ranked(case.blob, 4), eng.place_groups_lw(case.blob, rp),
            eng.place_groups_lw_ranked(case.blob, rp, 4), eng.place_groups_committed(case.blob))


def _same_outputs(x, y):
    for a, b in zip(x, y):
        a, b = (a,) if not isinstance(a, tuple) else a, (b,) if not isinstance(b, tuple) else b
        for u, v in zip(a, b):
            u, v = np.asarray(u), np.asarray(v)
            assert u.dtype == v.dtype and u.tobytes() == v.tobytes()


@pytest.mark.parametrize("seed,n", [(2, 31), (5, 2049)])
def test_reductions_and_existing_entry_points_unchanged(seed, n):
    case = gg.make_case(seed, n, scarce=seed % 2 == 0, exclusive=True)
    rp = cycle_pods(case.blob)
    full = full_masks(case.blob)
    eng = engine(case.topo)
    try:
        before = _outputs(eng, case, rp)
        eng.set_node_classes(random_classes(n, 5, seed), 5)
        _same_outputs(before, _outputs(eng, case, rp))   # installed classes change no existing entry point
        pg, pgr, plw, plwr, _ = before
        _same_outputs([pg], [eng.place_groups_eligible(case.blob, None, full)])
        _same_outputs([pgr], [eng.place_groups_eligible_ranked(case.blob, None, full, 4)])
        _same_outputs([plw], [eng.place_groups_eligible(case.blob, rp, full)])
        _same_outputs([plwr], [eng.place_groups_eligible_ranked(case.blob, rp, full, 4)])
        eng.set_node_classes(np.zeros(n, np.int32), 1)
        _same_outputs([plwr], [eng.place_groups_eligible_ranked(case.blob, rp, np.ones(len(full), np.uint64), 4)])
    finally:
        eng.close()


def _flat_topo(n, free=2, seed=4):
    topo = synth.make_topology(n, seed=seed, tiers=2, max_free=2)
    topo.domain_owner = np.full(int(topo.domain.max()) + 1, -1, np.int32)
    topo.free[:] = free
    return topo


@pytest.mark.parametrize("n,chunk", [(1, 0), (5, 0), (130, 0), (129, 128), (257, 128)])
def test_slab_edges(n, chunk):
    """N = 1, N % 4 != 0 (the slab's tail group), a one-node tail after chunks of 128; class 63 with bit 63; only node
    N - 1 admitted."""
    topo = _flat_topo(n)
    gblob = build([Group(gid=1, roles=[(0, 2, 1, 0), (0, 1, 1, 0)], pair=[[1, 1], [1, 1]]),
                   Group(gid=2, roles=[(0, 1, 1, 0)], pair=[[1]], flags=STEP_GANG)])
    eng = engine(topo, chunk_nodes=chunk)
    try:
        cls = np.zeros(n, np.int32)
        cls[-1] = 63
        eng.set_node_classes(cls, 64)
        for masks in ([1 << 63, 1 << 63, 1 << 63], [1 << 63, ALL, 1], [ALL, 1, 1 << 63]):
            got = check(eng, topo, gblob, None, np.asarray(masks, np.uint64), cls, 2)
            a = got[0]
            if masks[0] == 1 << 63:
                assert a[0] == n - 1
    finally:
        eng.close()


def _edgeless(n, free=1):
    z = np.zeros(0, np.int32)
    return dict(row_ptr=np.zeros(n + 1, np.int32), col_idx=z, edge_w=z, free=np.full(n, free, np.int32),
                domain=np.zeros(n, np.int32), domain_owner=np.full(1, -1, np.int32))


def test_large_fleets_and_the_room_bitmap_ceiling():
    """N = 2^20 + 1 with only the last node admitted; 1 638 400 nodes (the room bitmap's ceiling) places, one more is
    RBGTOPO_ELIMIT."""
    gblob = build([Group(gid=1, roles=[(0, 1, 1, 0), (0, 1, 1, 0)], pair=[[1, 0], [0, 1]])])
    for n, code in ((2 ** 20 + 1, 0), (1_638_400, 0), (1_638_401, -6)):
        t = _edgeless(n)
        eng = TopoPlacer(device=0)
        try:
            eng.set_topology(t["row_ptr"], t["col_idx"], t["edge_w"], t["free"], t["domain"], t["domain_owner"])
            cls = np.zeros(n, np.int32)
            cls[-1] = 1
            eng.set_node_classes(cls, 2)
            masks = np.asarray([0b10, 0b01], np.uint64)
            if code:
                assert _code(lambda: eng.place_groups_eligible(gblob, None, masks)) == code
                continue
            a, s, d, sc, an, asc = eng.place_groups_eligible_ranked(gblob, None, masks, 2)
            assert a[0] == n - 1 and a[1] == 0 and s.tolist() == [0]   # equal rows: node order breaks the tie
            assert (an[0] == -1).all() and an[1].tolist() == [1, 2]
        finally:
            eng.close()


def test_classes_issued_behind_an_in_flight_call_and_dropped_by_set_topology():
    """set_node_classes issued while the caller stream still runs earlier work returns without waiting for it, and
    the next call sees the new classes; a call made before it keeps the old ones."""
    import torch
    from gpu_util import SLEEP_CYCLES, sleep_on
    case = gg.make_case(3, 130, scarce=False, exclusive=True)
    n = 130
    rp = cycle_pods(case.blob)
    cls_a, cls_b = random_classes(n, 3, 1), random_classes(n, 3, 2)
    masks = random_masks(case.blob, 3, 7)
    st = torch.cuda.Stream()
    eng = engine(case.topo)
    try:
        eng.set_stream(st.cuda_stream)
        eng.set_node_classes(cls_a, 3)
        sleep_on(st)
        got_a = eng.place_groups_eligible(case.blob, rp, masks)   # waits behind the sleep, reads cls_a
        sleep_on(st, 4 * SLEEP_CYCLES)
        eng.set_node_classes(cls_b, 3)   # ordered behind the pending sleep on the refresh stream, not waited for
        assert not st.query()
        got_b = eng.place_groups_eligible(case.blob, rp, masks)
        torch.cuda.synchronize()
        same_a = run_eligible(case.topo, case.blob, rp, masks, cls_a)
        same_b = run_eligible(case.topo, case.blob, rp, masks, cls_b)
        for x, y in zip(got_a, same_a):
            assert np.array_equal(x, y)
        for x, y in zip(got_b, same_b):
            assert np.array_equal(x, y)
        eng.set_topology(case.topo.row_ptr, case.topo.col_idx, case.topo.edge_w, case.topo.free, case.topo.domain,
                         case.topo.domain_owner)
        assert _code(lambda: eng.place_groups_eligible(case.blob, rp, masks)) == -1
        eng.set_node_classes(cls_b, 3)
        for x, y in zip(eng.place_groups_eligible(case.blob, rp, masks), same_b):
            assert np.array_equal(x, y)
    finally:
        eng.close()


def test_error_codes_and_recovery():
    case = gg.make_case(2, 31, scarce=True, exclusive=True)
    n = 31
    rp = cycle_pods(case.blob)
    masks = full_masks(case.blob)
    fresh = TopoPlacer(device=0)
    try:
        assert _code(lambda: fresh.set_node_classes(np.zeros(n, np.int32), 1)) == -5
    finally:
        fresh.close()
    eng = engine(case.topo)
    try:
        assert _code(lambda: eng.place_groups_eligible(case.blob, rp, masks)) == -1          # no classes installed
        assert _code(lambda: eng.set_node_classes(np.zeros(n, np.int32), 65)) == -6
        assert _code(lambda: eng.set_node_classes(np.zeros(n, np.int32), 0)) == -1
        assert _code(lambda: eng.set_node_classes(np.full(n, 3, np.int32), 3)) == -1
        assert _code(lambda: eng.set_node_classes(np.full(n, -1, np.int32), 3)) == -1
        cls = random_classes(n, 3, 0)
        eng.set_node_classes(cls, 3)
        assert _code(lambda: eng.place_groups_eligible(case.blob, rp, masks[:-1])) == -1     # one mask short
        assert _code(lambda: eng.place_groups_eligible(case.blob, None, np.append(masks, np.uint64(1)))) == -1
        assert _code(lambda: eng.place_groups_eligible(case.blob, rp[:-1], masks)) == -1     # role_pods short
        assert _code(lambda: eng.place_groups_eligible_ranked(case.blob, rp, masks, 9)) == -1
        assert _code(lambda: eng.place_groups_eligible(case.blob[:-1], rp, masks)) == -1
        check(eng, case.topo, case.blob, rp, random_masks(case.blob, 3, 1), cls, 2)         # still usable
    finally:
        eng.close()
    from rbg_b200 import _lib
    engs = [engine(case.topo, rank=r, world=2, lw_shards=True) for r in range(2)]
    try:
        gb, rpa = np.ascontiguousarray(case.blob, np.int32), np.ascontiguousarray(np.asarray(rp).reshape(-1), np.int32)
        mk = np.ascontiguousarray(masks, np.uint64)
        for e in engs:
            e.set_node_classes(np.zeros(n, np.int32), 1)
            assert not e.places_eligible
            outs = [np.full(4096, 12345, np.int32) for _ in range(3)]
            ptr = [o.ctypes.data_as(_lib.i32p) for o in outs]
            rc = e.lib.rbgtopo_place_groups_eligible(e._h, gb.ctypes.data_as(_lib.i32p), len(gb),
                                                     rpa.ctypes.data_as(_lib.i32p), len(rpa),
                                                     mk.ctypes.data_as(_lib.u64p), len(mk), *ptr)
            assert rc == -6 and all((o == 12345).all() for o in outs)   # refused before anything is written
            e.place_groups_lw(case.blob, rp)
    finally:
        for e in engs:
            e.close()
