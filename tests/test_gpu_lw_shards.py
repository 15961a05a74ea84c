"""GPU: leader-worker placement on node-axis shards (DESIGN.md §3.18) with world = 1, 2 and 4 contexts on one device.
rbgtopo_place_groups_lw / _lw_committed on a ctx with RBGTOPO_CFG_LW_SHARDS, and the sharded ranked forms
rbgtopo_shard_place_groups_lw[_committed]_ranked + rbgtopo_shard_alternates_merge, whose all-gather is a device
concatenation of the ranks' exchange buffers, rank-major (what the NCCL all-gather produces between GPUs; on >= 2 GPUs
a torch.distributed.run worker repeats the plain and committed cases over NCCL).  On every rank every output is
compared bit for bit with the world = 1 call on the same snapshot, which the existing suites hold to the oracles."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import groups_gen as gg
import lw_commit_gen as lg
import lw_commit_levels_gen as lvg
import lw_oracle as lw
from rbg_b200 import _lib, synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, STEP_GANG, Group, GroupsBuilder
from rbg_b200.engine import RbgTopoError, TopoPlacer
from test_gpu_shard_alternates import bits, close, code, gather

pytestmark = pytest.mark.gpu

EINVAL, EINEXACT, ELIMIT = -1, -4, -6
HERE = os.path.dirname(os.path.abspath(__file__))


def engines(topo, world, setup=None, **kw):
    engs = []
    for r in range(world):
        e = TopoPlacer(device=0, rank=r, world=world, **kw)
        e.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
        if setup:
            setup(e)
        engs.append(e)
    return engs


def same(got, exp, what):
    assert len(got) == len(exp), what
    for i, (x, y) in enumerate(zip(got, exp)):
        if isinstance(y, (int, np.integer)):
            assert int(x) == int(y), (what, i, x, y)
        else:
            assert np.array_equal(bits(x), bits(y)), (what, i, np.nonzero(bits(x) != bits(y))[0][:8])


def place(e, gb, rp, committed):
    return e.place_groups_lw_committed(gb, rp) if committed else e.place_groups_lw(gb, rp)


def ranked(e, gb, rp, n_alt, committed):
    return e.place_groups_lw_committed_ranked(gb, rp, n_alt) if committed else e.place_groups_lw_ranked(gb, rp, n_alt)


def sharded(engs, gb, rp, n_alt, committed=False):
    """Both halves on every rank: (per-rank outputs in the world = 1 ranked call's layout, keys_bytes per rank)."""
    locs = [e.shard_place_groups_lw_committed_ranked(gb, rp, n_alt) if committed
            else e.shard_place_groups_lw_ranked(gb, rp, n_alt) for e in engs]
    allk = gather([(l[-2], l[-1]) for l in locs])
    outs = []
    for e, l in zip(engs, locs):
        placed = l[:-3]
        outs.append((*placed, *e.shard_alternates_merge(l[-3], allk.data_ptr(), len(placed[0]), n_alt)))
    return outs, [l[-1] for l in locs]


def check_worlds(topo, gb, rp, committed=False, n_alts=(0, 4, 8), worlds=(2, 4), setup=None, **kw):
    """World = 1 (flag-less and with the flag) against every rank of every world: the unranked call on a ctx with
    RBGTOPO_CFG_LW_SHARDS and the sharded ranked form on a ctx without it."""
    e1 = engines(topo, 1, setup, **kw)[0]
    ef = engines(topo, 1, setup, lw_shards=True, **kw)[0]
    try:
        ref = place(e1, gb, rp, committed)
        same(place(ef, gb, rp, committed), ref, "the flag at world 1")
        refs = {F: ranked(e1, gb, rp, F, committed) for F in n_alts}
        for F in n_alts:
            outs, _ = sharded([e1], gb, rp, F, committed)
            same(outs[0], refs[F], ("sharded ranked at world 1", F))
    finally:
        close([e1, ef])
    for W in worlds:
        engs = engines(topo, W, setup, lw_shards=True, **kw)
        try:
            for r, e in enumerate(engs):
                same(place(e, gb, rp, committed), ref, (W, r))
            for F in n_alts:
                outs, nbytes = sharded(engs, gb, rp, F, committed)
                assert len(set(nbytes)) == 1, nbytes
                assert nbytes[0] % 8 == 0 and nbytes[0] >= 8, nbytes   # 72 per job + 4 per placed pod, padded
                for r, o in enumerate(outs):
                    same(o, refs[F], (W, r, F))
        finally:
            close(engs)
    return ref, refs


def cycle_pods(gblob, S=(2, 4, 1), C=(-1, 0)):
    k = iter(range(1 << 20))
    return lw.role_pods_for(gblob, lambda g, r: (S[(g + r) % len(S)], C[next(k) % len(C)]))


# ---- rbgtopo_place_groups_lw and its ranked form

@pytest.mark.parametrize("seed,n,scarce,excl", gg.CASES)
def test_generated_fleets(seed, n, scarce, excl):
    case = gg.make_case(seed, n, scarce=scarce, exclusive=excl)
    ref, _ = check_worlds(case.topo, case.blob, cycle_pods(case.blob), n_alts=(0, 8))
    exp = lw.run_lw(case.topo, case.blob, cycle_pods(case.blob))
    same(ref, exp, "oracle")


def test_full_32_pod_waves_demand_0_gang_and_anchors():
    n = 130
    topo = synth.make_topology(n, seed=9, tiers=3, max_free=3)
    topo.domain_owner[:] = -1
    rng = np.random.default_rng(9)
    gb = lg.build([
        Group(gid=1, roles=[(0, 3, 0, 0)], pair=[[1]]),                                    # demand 0, S = 32
        Group(gid=2, roles=[(0, 2, 1, 0), (0, 3, 1, 0), (1, 2, 2, 0)], pair=[[1, 1, 1], [1, 1, 0], [1, 0, 2]],
              anchors=[(int(x), int(rng.integers(0, 3)), 2) for x in rng.choice(n, 5, replace=False)]),
        Group(gid=3, roles=[(0, 6, 2, 0)], pair=[[1]], flags=STEP_GANG),                   # gang that cannot fit
        Group(gid=4, roles=[(0, 2, 1, 0)], pair=[[1]], flags=STEP_GANG),                   # gang that fits
    ])
    for rp in ([(32, -1), (2, 0), (5, -1), (1, 0), (32, 0), (3, 0)],
               [(32, 0), (1, -1), (4, 0), (3, -1), (16, -1), (2, -1)]):
        ref, _ = check_worlds(topo, gb, rp)
        assert 2 in ref[1].tolist() and 0 in ref[1].tolist()


@pytest.mark.parametrize("seed,n", [(1, 33), (3, 2049)])
def test_colocation_at_every_level_and_exclusive_levels(seed, n):
    """Levels 1 (one domain per node) and 2 (racks of 16) installed, exclusive groups at levels 0 and 2, C in
    {-1, 0, 1, 2}, on a ctx with RBGTOPO_CFG_LEVEL_PLACEMENT."""
    topo = synth.make_topology(n, seed=seed, tiers=2, max_free=4)
    topo.domain_owner[:] = -1
    lv = [topo.domain, np.arange(n, dtype=np.int32), (np.arange(n) // 16).astype(np.int32)]
    rng = np.random.default_rng(seed)
    groups = []
    for g in range(12):
        L = (0, 2, 0, 2)[g % 4] if g % 3 else 0
        excl = g % 3 != 1
        fixed = int(rng.integers(0, int(lv[L].max()) + 1)) if excl and g % 5 == 0 else -1
        roles = [(0, int(rng.integers(1, 4)), int(rng.integers(0, 3)), ROLE_EXCLUSIVE),
                 (0, int(rng.integers(0, 3)), 1, ROLE_EXCLUSIVE if g % 2 else 0),
                 (1, int(rng.integers(1, 3)), 1, ROLE_EXCLUSIVE)]
        groups.append(Group(gid=10 + g, roles=roles, pair=[[1, 1, 0], [1, 1, 1], [0, 1, 1]],
                            anchors=[(int(rng.integers(0, n)), 0, 1)],
                            flags=(STEP_EXCLUSIVE if excl else 0) | (STEP_GANG if g % 4 == 3 else 0),
                            fixed_domain=fixed, level=L))
    gb = lg.build(groups)
    rp = lw.role_pods_for(gb, lambda g, r: ((2, 3, 4)[(g + r) % 3], (0, 1, 2, -1)[(g + 2 * r) % 4]))
    setup = lambda e: e.set_exclusive_levels(lv[1:], np.zeros((0, 3), np.int32))
    ref, _ = check_worlds(topo, gb, rp, setup=setup, level_placement=True)
    assert (ref[2] >= 0).any() and (ref[0] >= 0).any()


def slab_topology():
    """Domains of 100 nodes on 1 000 nodes: at world 2 the slab bound is 384, inside domain 3."""
    n = 1000
    topo = synth.make_topology(n, seed=2, tiers=2, max_free=3)
    topo.domain = (np.arange(n) // 100).astype(np.int32)
    topo.domain_owner = np.full(10, -1, np.int32)
    return topo


def test_domains_that_straddle_a_slab_bound():
    """Exclusive groups fixed to domain 3 and co-located in level-0 domains, which hold nodes of both slabs."""
    topo = slab_topology()
    b = GroupsBuilder()
    for i in range(6):
        b.add(Group(gid=10 + i, roles=[(0, 3 + i, 1, ROLE_EXCLUSIVE), (1, 2, 1, 0)], pair=[[1, 1], [1, 1]],
                    anchors=[(380 + i, 0, 1)], flags=STEP_EXCLUSIVE, fixed_domain=3 if i < 4 else -1))
    gb = b.build()
    for rp in ([(2, 0), (3, -1)] * 6, [(4, 0), (2, 0)] * 6):
        ref, _ = check_worlds(topo, gb, rp)
        assert (ref[0] >= 0).any()


def test_a_d_star_whose_best_node_lies_in_another_slab():
    """Only nodes >= 400 have room, so the best node of the first participating row lies in rank 1's slab at world 2
    (bound 384) and in rank 3's at world 4: the other ranks find D* outside their slabs."""
    topo = slab_topology()
    topo.free[:400] = 0
    gb = lg.build([Group(gid=5, roles=[(0, 2, 1, ROLE_EXCLUSIVE), (1, 2, 1, ROLE_EXCLUSIVE)], pair=[[1, 1], [1, 1]],
                         anchors=[(917, 0, 3)], flags=STEP_EXCLUSIVE)])
    ref, _ = check_worlds(topo, gb, [(2, -1), (2, 0)])
    assert ref[2][0] >= 4 and (ref[0] >= 400).all(), ref


def test_groups_the_host_loop_re_runs_and_failed_gangs():
    """Non-gang groups with unplaced replicas reach later waves with fewer anchors; gangs fail as a whole."""
    topo = synth.make_topology(300, seed=5, tiers=2, max_free=2)
    topo.domain_owner[:] = -1
    topo.free = np.where(np.arange(300) % 3 == 0, 0, topo.free).astype(np.int32)
    gb = lg.build([Group(gid=1 + g, roles=[(0, 4, 2, 0), (1, 3, 1, 0), (2, 2, 1, 0)],
                         pair=[[1, 1, 0], [1, 2, 1], [0, 1, 1]], flags=STEP_GANG if g % 2 else 0) for g in range(8)])
    ref, _ = check_worlds(topo, gb, [(8, 0), (4, -1), (2, 0)] * 8)
    assert 1 in ref[1].tolist() and 2 in ref[1].tolist(), ref[1]


# ---- committed batches

@pytest.mark.parametrize("seed,n,scarce", lg.SEEDS)
@pytest.mark.parametrize("mode", ["map", "occupancy"])
def test_committed_batches(seed, n, scarce, mode):
    occ = mode == "occupancy"
    f = lg.fleet(seed, n, n_groups=14, scarce=scarce, levels=occ, occupancy=occ)
    setup = (lambda e: e.set_exclusive_levels(f.lv[1:], f.occ)) if occ else None
    check_worlds(f.topo, f.blob(), f.role_pods(), committed=True, n_alts=(0, 8), setup=setup)


@pytest.mark.parametrize("seed,n,scarce,kind", lvg.SEEDS)
def test_committed_batches_at_levels(seed, n, scarce, kind):
    """Flags 15: committed leader-worker batches at every exclusive level on node-axis shards."""
    f = lvg.fleet(seed, n, n_groups=14, scarce=scarce, kind=kind)
    setup = lambda e: e.set_exclusive_levels(f.lv[1:], f.occ)
    ref, _ = check_worlds(f.topo, f.blob(), f.role_pods(), committed=True, n_alts=(0, 4), setup=setup,
                          lw_committed_levels=True)
    same(ref[:3], f.expected(), "oracle")


# ---- checks: those of world 1, nothing written

def raw_lw(e, gb, rp, committed, assign):
    rounds = C.c_int32(9)
    i32 = _lib.i32p
    if committed:
        rc = e.lib.rbgtopo_place_groups_lw_committed(e._h, gb.ctypes.data_as(i32), len(gb), rp.ctypes.data_as(i32),
                                                     len(rp), assign.ctypes.data_as(i32), None, None, C.byref(rounds))
    else:
        rc = e.lib.rbgtopo_place_groups_lw(e._h, gb.ctypes.data_as(i32), len(gb), rp.ctypes.data_as(i32), len(rp),
                                           assign.ctypes.data_as(i32), None, None)
    return rc, rounds.value


def raw_local(e, gb, rp, n_alt, committed, assign):
    xh, p, nb, rounds = C.c_int32(-7), C.c_void_p(0), C.c_int64(-7), C.c_int32(9)
    i32 = _lib.i32p
    args = (e._h, gb.ctypes.data_as(i32), len(gb), rp.ctypes.data_as(i32), len(rp), n_alt, assign.ctypes.data_as(i32),
            None, None)
    if committed:
        rc = e.lib.rbgtopo_shard_place_groups_lw_committed_ranked(*args, C.byref(rounds), C.byref(xh), C.byref(p),
                                                                  C.byref(nb))
    else:
        rc = e.lib.rbgtopo_shard_place_groups_lw_ranked(*args, C.byref(xh), C.byref(p), C.byref(nb))
    return rc, xh.value, p.value, nb.value, rounds.value


def check_refused(topo, gb, rp, expect=None, committed=False, n_alt=8, setup=None, **kw):
    """The world = 1 code on every rank of worlds 1 and 2, for the unranked call on a ctx with the flag and for the
    sharded ranked local half, with nothing written."""
    rp = np.ascontiguousarray(np.asarray(rp, dtype=np.int32).reshape(-1))
    e1 = engines(topo, 1, setup, **kw)[0]
    try:
        c1 = code(lambda: place(e1, gb, rp, committed))   # 0 when only n_alt is wrong
        c2 = code(lambda: ranked(e1, gb, rp, n_alt, committed))
    finally:
        e1.close()
    assert c2 != 0 and (expect is None or c2 == expect), (c2, expect)
    for W in (1, 2):
        engs = engines(topo, W, setup, lw_shards=True, **kw)
        try:
            for e in engs:
                assign = np.full(4096, 12345, np.int32)
                if c1:
                    rc, rounds = raw_lw(e, gb, rp, committed, assign)
                    assert rc == c1 and (assign == 12345).all(), (W, rc, c1)
                    assert rounds == (0 if committed else 9)
                rc, xh, p, nb, rounds = raw_local(e, gb, rp, n_alt, committed, assign)
                assert rc == c2, (W, rc, c2)
                assert (assign == 12345).all() and xh == -7 and not p and nb == -7, (W, xh, p, nb)
        finally:
            close(engs)


def test_errors_are_those_of_world_1_with_nothing_written():
    case = gg.make_case(3, 33, exclusive=True)
    gb, rp = case.blob, cycle_pods(case.blob)
    for committed in (False, True):
        check_refused(case.topo, gb, rp, EINVAL, committed, n_alt=9)
        check_refused(case.topo, gb, rp[:-1], EINVAL, committed)                      # role_pods too short
        bad = rp.copy()
        bad[0] = (33, -1)
        check_refused(case.topo, gb, bad, EINVAL, committed)                          # S above 32
        bad[0] = (2, 5)
        check_refused(case.topo, gb, bad, EINVAL, committed)                          # C above the installed levels
        for word, value in [(0, 0), (2, -1), (8 + 3, 0), (8 + 3, 17), (8 + 10, 1)]:
            b = gb.copy()
            b[word] = value
            check_refused(case.topo, b, rp, None, committed)


def test_without_the_flag_world_2_keeps_elimit():
    case = gg.make_case(2, 33)
    gb, rp = case.blob, cycle_pods(case.blob)
    engs = engines(case.topo, 2)
    try:
        for e in engs:
            assert not e.places_lw_sharded
            for fn in (lambda: e.place_groups_lw(gb, rp), lambda: e.place_groups_lw_committed(gb, rp),
                       lambda: e.place_groups_lw_ranked(gb, rp, 4), lambda: e.place_groups_lw_committed_ranked(gb, rp, 4)):
                assert code(fn) == ELIMIT
    finally:
        close(engs)
    engs = engines(case.topo, 2, lw_shards=True)
    try:
        for e in engs:
            assert e.places_lw_sharded
            assert code(lambda: e.place_groups_lw_ranked(gb, rp, 4)) == ELIMIT
            assert code(lambda: e.place_groups_lw_committed_ranked(gb, rp, 4)) == ELIMIT
    finally:
        close(engs)


def test_exactness_bound_is_that_of_world_1():
    topo = synth.make_topology(256, seed=3, tiers=2, max_free=2)
    blob = lambda A: GroupsBuilder().add(Group(gid=1, roles=[(0, 6, 1, 0)], pair=[[1]], anchors=[(7, 0, A)],
                                               flags=0)).build()
    rp = [(4, 0)]
    e1 = TopoPlacer(device=0)
    e1.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    try:
        lo_, hi = 1, 1 << 20   # the largest anchor count the call accepts
        while hi - lo_ > 1:
            mid = (lo_ + hi) // 2
            if code(lambda: e1.place_groups_lw(blob(mid), rp)) == 0:
                lo_ = mid
            else:
                hi = mid
        assert code(lambda: e1.place_groups_lw(blob(lo_ + 1), rp)) == EINEXACT
    finally:
        e1.close()
    for committed in (False, True):
        check_refused(topo, blob(lo_ + 1), rp, EINEXACT, committed, n_alt=0)
        check_worlds(topo, blob(lo_), rp, committed=committed, n_alts=(8,), worlds=(2,))


def test_room_bitmap_limit_is_on_n():
    """N = 1 638 401 at world 2: ELIMIT, though each slab would fit; N = 1 638 400 is placed and ranked."""
    def topo_of(n):
        rp = (2 * np.arange(n + 1)).astype(np.int32)   # a ring
        col = np.sort(np.stack([(np.arange(n) - 1) % n, (np.arange(n) + 1) % n], axis=1), axis=1).ravel().astype(np.int32)
        free = np.ones(n, np.int32)
        free[::7] = 2
        return synth.Topology(rp, col, np.ones(2 * n, np.int32), free, (np.arange(n) // 4096).astype(np.int32),
                              np.full((n + 4095) // 4096, -1, np.int32))
    b = GroupsBuilder()
    b.add(Group(gid=1, roles=[(0, 3, 1, 0), (1, 2, 2, 0)], pair=[[1, 1], [1, 1]], anchors=[(5, 0, 1)], flags=0))
    b.add(Group(gid=2, roles=[(0, 4, 1, 0)], pair=[[1]], anchors=[(1638399, 0, 2)], flags=0))
    gb = b.build()
    rp = [(2, 0), (1, -1), (3, -1)]
    big = 200 * 1024 * 8
    for committed in (False, True):
        check_refused(topo_of(big + 1), gb, rp, ELIMIT, committed)
        check_worlds(topo_of(big), gb, rp, committed=committed, n_alts=(8,), worlds=(2,))


def test_refresh_release_double_merge_and_the_other_entry_points():
    case = gg.make_case(6, 4097, scarce=True, exclusive=True)
    topo, gb = case.topo, case.blob
    rp = cycle_pods(gb, S=(2, 1, 3))
    free2 = np.maximum(topo.free - 1, 0).astype(np.int32)
    e1 = engines(topo, 1)[0]
    try:
        ref, cref = e1.place_groups_lw(gb, rp), e1.place_groups_lw_committed(gb, rp)
        rref, crref = e1.place_groups_lw_ranked(gb, rp, 8), e1.place_groups_lw_committed_ranked(gb, rp, 8)
        groups, committed = e1.place_groups(gb), e1.place_groups_committed(gb)
        e1.update_nodes(free=free2)
        ref2 = e1.place_groups_lw(gb, rp)
    finally:
        e1.close()
    engs = engines(topo, 2, lw_shards=True)
    try:
        P = len(ref[0])
        la = [e.shard_place_groups_lw_ranked(gb, rp, 8) for e in engs]
        lb = [e.shard_place_groups_lw_committed_ranked(gb, rp, 8) for e in engs]
        for e in engs:   # a refresh between the halves changes no merge
            e.update_nodes(free=free2)
        ka, kb = gather([(l[-2], l[-1]) for l in la]), gather([(l[-2], l[-1]) for l in lb])
        for e, l in zip(engs, lb):
            same((*l[:4], *e.shard_alternates_merge(l[-3], kb.data_ptr(), P, 8)), crref, "committed, second")
        for e, l in zip(engs, la):
            same((*l[:3], *e.shard_alternates_merge(l[-3], ka.data_ptr(), P, 8)), rref, "first")
            assert code(lambda: e.shard_alternates_merge(l[-3], ka.data_ptr(), P, 8)) == EINVAL   # consumed
        for e in engs:   # the refreshed snapshot places as world 1 does
            same(e.place_groups_lw(gb, rp), ref2, "after update_nodes")
            e.update_nodes(free=topo.free)
            l = e.shard_place_groups_lw_ranked(gb, rp, 8)
            e.release(l[-3])
            assert code(lambda: e.shard_alternates_merge(l[-3], ka.data_ptr(), P, 8)) == EINVAL
        for e in engs:   # the other entry points afterwards, and these calls again
            same(e.place_groups(gb), groups, "place_groups")
            same(e.place_groups_committed(gb), committed, "place_groups_committed")
            same(e.place_groups_lw(gb, rp), ref, "place_groups_lw again")
            same(e.place_groups_lw_committed(gb, rp), cref, "place_groups_lw_committed again")
        outs, _ = sharded(engs, gb, rp, 8)
        for o in outs:
            same(o, rref, "ranked again")
    finally:
        close(engs)


def test_high_level_methods_at_world_1():
    case = gg.make_case(4, 130, scarce=True, exclusive=True)
    rp = cycle_pods(case.blob)
    e1 = engines(case.topo, 1)[0]
    try:
        same(e1.place_groups_lw_ranked_sharded(case.blob, rp, 8), e1.place_groups_lw_ranked(case.blob, rp, 8), "w1")
        same(e1.place_groups_lw_committed_ranked_sharded(case.blob, rp, 8),
             e1.place_groups_lw_committed_ranked(case.blob, rp, 8), "w1 committed")
    finally:
        e1.close()


WORKER = r'''
import os, sys
import numpy as np, torch, torch.distributed as dist
sys.path.insert(0, os.environ["RBG_ROOT"]); sys.path.insert(0, os.path.join(os.environ["RBG_ROOT"], "tests"))
import groups_gen as gg
import lw_commit_gen as lg
import lw_oracle as lw
from rbg_b200.engine import TopoPlacer
rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
def eng_of(topo, w, r, **kw):
    e = TopoPlacer(device=local, rank=r, world=w, **kw)
    e.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    return e
def bits(x):
    x = np.asarray(x)
    return x.view(np.uint32) if x.dtype == np.float32 else x
cases = []
for s, n, sc, ex in gg.CASES[:6]:
    c = gg.make_case(s, n, scarce=sc, exclusive=ex)
    cases.append((c.topo, c.blob, lw.role_pods_for(c.blob, lambda g, r: ((2, 4, 1)[(g + r) % 3], (-1, 0)[r % 2])), False))
for s, n, sc in lg.SEEDS[:4]:
    f = lg.fleet(s, n, n_groups=14, scarce=sc)
    cases.append((f.topo, f.blob(), f.role_pods(), True))
for topo, gb, rp, committed in cases:
    e1, e = eng_of(topo, 1, 0), eng_of(topo, world, rank, lw_shards=True)
    ref = e1.place_groups_lw_committed(gb, rp) if committed else e1.place_groups_lw(gb, rp)
    got = e.place_groups_lw_committed(gb, rp) if committed else e.place_groups_lw(gb, rp)
    for x, y in zip(got, ref):
        assert np.array_equal(bits(x), bits(y)), (rank, committed)
    for n_alt in (0, 8):
        if committed:
            ref, got = e1.place_groups_lw_committed_ranked(gb, rp, n_alt), e.place_groups_lw_committed_ranked_sharded(gb, rp, n_alt)
        else:
            ref, got = e1.place_groups_lw_ranked(gb, rp, n_alt), e.place_groups_lw_ranked_sharded(gb, rp, n_alt)
        for x, y in zip(got, ref):
            assert np.array_equal(bits(x), bits(y)), (rank, committed, n_alt)
    e1.close(); e.close()
dist.barrier()
if rank == 0: print("LW_SHARDS_OK", world)
dist.destroy_process_group()
'''


def test_plain_and_committed_over_nccl(tmp_path):
    import torch
    ngpu = torch.cuda.device_count()
    if ngpu < 2:
        pytest.skip("one GPU: NCCL needs one device per rank; the cases above run the ranks as contexts of this device")
    world = 2 if ngpu < 4 else 4
    script = tmp_path / "lw_shards_worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, RBG_ROOT=os.path.dirname(HERE))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
                        "--master-addr", "127.0.0.1", "--master-port", "29521", str(script)],
                       env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "LW_SHARDS_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
