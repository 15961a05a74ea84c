"""GPU: ranked alternates on node-axis shards (rbgtopo_shard_place_groups*_ranked + rbgtopo_shard_alternates_merge,
DESIGN.md §3.17) with world = 1, 2 and 4 contexts on one device.  The all-gather is a device concatenation of the
ranks' exchange buffers, rank-major, which is what the NCCL all-gather produces between GPUs (on >= 2 GPUs a
torch.distributed.run worker repeats the plain and committed cases over NCCL).  On every rank every output is
compared bit for bit with the world = 1 place_groups_ranked / place_groups_committed_ranked on the same snapshot,
which the existing suites hold to the oracle; the plain fleets are also checked against the oracle here."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import commit_gen as cg
import commit_levels_gen as clg
import committed_alternates_oracle as cao
import groups_gen as gg
import levels_oracle as lo
from alternates_oracle import run_fleet_ranked
from oracle import wave_loop
from rbg_b200 import _lib, synth
from rbg_b200.blob import Group, GroupsBuilder
from rbg_b200.engine import RbgTopoError, TopoPlacer

pytestmark = pytest.mark.gpu

EINVAL, EINEXACT, ELIMIT = -1, -4, -6
HERE = os.path.dirname(os.path.abspath(__file__))


class DevPtr:
    def __init__(self, p, nb):
        self.__cuda_array_interface__ = {"shape": (nb,), "typestr": "|u1", "data": (p, False), "version": 3,
                                         "strides": None}


def gather(bufs):
    """All-gather of one exchange buffer per rank on a single GPU: concatenate, rank-major."""
    import torch
    torch.cuda.synchronize()
    out = torch.cat([torch.as_tensor(DevPtr(p, nb), device="cuda") for p, nb in bufs])
    torch.cuda.synchronize()
    return out


def engines(topo, world, **kw):
    engs = []
    for r in range(world):
        e = TopoPlacer(device=0, rank=r, world=world, **kw)
        e.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
        engs.append(e)
    return engs


def close(engs):
    for e in engs:
        e.close()


def bits(x):
    x = np.asarray(x)
    return x.view(np.uint32) if x.dtype == np.float32 else x


def same(got, exp, what):
    assert len(got) == len(exp), what
    for i, (x, y) in enumerate(zip(got, exp)):
        if isinstance(y, (int, np.integer)):
            assert int(x) == int(y), (what, i, x, y)
        else:
            assert np.array_equal(bits(x), bits(y)), (what, i, np.nonzero(bits(x) != bits(y))[0][:8])


def local(e, gb, n_alt, committed):
    return e.shard_place_groups_committed_ranked(gb, n_alt) if committed else e.shard_place_groups_ranked(gb, n_alt)


def sharded(engs, gb, n_alt, committed=False):
    """Both halves on every rank: (per-rank outputs in the world = 1 call's layout, keys_bytes per rank)."""
    locs = [local(e, gb, n_alt, committed) for e in engs]
    allk = gather([(l[-2], l[-1]) for l in locs])
    outs = []
    for e, l in zip(engs, locs):
        placed = l[:-3]
        outs.append((*placed, *e.shard_alternates_merge(l[-3], allk.data_ptr(), len(placed[0]), n_alt)))
    return outs, [l[-1] for l in locs]


def world1(e1, gb, n_alt, committed=False):
    return e1.place_groups_committed_ranked(gb, n_alt) if committed else e1.place_groups_ranked(gb, n_alt)


def check_worlds(topo, gb, n_alts=(0, 8), committed=False, worlds=(1, 2, 4), setup=None, **kw):
    """Every world and n_alt against the world = 1 ranked call on a ctx with the same flags and snapshot."""
    e1 = TopoPlacer(device=0, **kw)
    e1.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    if setup:
        setup(e1)
    refs = {F: world1(e1, gb, F, committed) for F in n_alts}
    e1.close()
    for W in worlds:
        engs = engines(topo, W, **kw)
        try:
            for e in engs:
                if setup:
                    setup(e)
            for F in n_alts:
                outs, nbytes = sharded(engs, gb, F, committed)
                assert len(set(nbytes)) == 1, nbytes
                for r, o in enumerate(outs):
                    same(o, refs[F], (W, r, F))
        finally:
            close(engs)
    return refs


# ---- fleets

@pytest.mark.parametrize("seed,n,scarce,excl", gg.CASES)
def test_generated_fleets(seed, n, scarce, excl):
    case = gg.make_case(seed, n, scarce=scarce, exclusive=excl)
    refs = check_worlds(case.topo, case.blob)
    exp = run_fleet_ranked(case.topo, wave_loop.groups_from_blob(case.blob), 8)
    same(refs[8], exp, "oracle")


def test_exclusive_domains_across_a_slab_boundary():
    """Domains of 100 nodes on 1 000 nodes: at world 2 the slab bound is 384, inside domain 3; exclusive groups fixed
    to domain 3 rank nodes of both slabs."""
    n = 1000
    topo = synth.make_topology(n, seed=2, tiers=2, max_free=3)
    topo.domain = (np.arange(n) // 100).astype(np.int32)
    topo.domain_owner = np.full(10, -1, np.int32)
    b = GroupsBuilder()
    for i in range(6):
        fixed = 3 if i < 4 else -1
        b.add(Group(gid=10 + i, roles=[(0, 3 + i, 1, 1), (1, 2, 1, 0)], pair=[[1, 1], [1, 1]], anchors=[],
                    flags=1, fixed_domain=fixed))
    gb = b.build()
    refs = check_worlds(topo, gb, n_alts=(8,))
    exp = run_fleet_ranked(topo, wave_loop.groups_from_blob(gb), 8)
    same(refs[8], exp, "oracle")
    alts = refs[8][4]
    assert ((alts >= 300) & (alts < 384)).any() and ((alts >= 384) & (alts < 400)).any(), alts


def test_groups_the_host_loop_re_runs_and_failed_gangs():
    from test_gpu_alternates import rerun_case
    for seed in range(3):
        topo, gb = rerun_case(seed)
        refs = check_worlds(topo, gb, n_alts=(0, 4, 8))
        s = refs[8][1]
        assert (s == 1).any() and (s == 2).any(), s
        same(refs[8], run_fleet_ranked(topo, wave_loop.groups_from_blob(gb), 8), "oracle")


@pytest.mark.parametrize("seed,n,kind", [(42, 33, "mixed"), (43, 33, "random"), (45, 2049, "random")])
def test_levels_on_a_level_placement_ctx(seed, n, kind):
    from test_gpu_levels_place import fleet
    topo, lv, nd, gb, occ = fleet(seed, n, kind, scarce=seed % 2 == 0)
    check_worlds(topo, gb, setup=lambda e: e.set_exclusive_levels(lv[1:], occ, level_n_domains=nd[1:]),
                 level_placement=True, chunk_nodes=128)


@pytest.mark.parametrize("i", range(0, len(cg.cases()), 3))
def test_committed_batches(i):
    case = cg.cases()[i]
    refs = check_worlds(case.topo, case.blob, committed=True)
    exp = cao.run_fleet_committed_ranked(case.topo, wave_loop.groups_from_blob(case.blob), 8, fast=True)
    same((refs[8][0], refs[8][1], refs[8][2], refs[8][4], refs[8][5], refs[8][6]), exp, "oracle")


@pytest.mark.parametrize("i", range(0, len(clg.cases()), 2))
def test_committed_batches_at_levels(i):
    c = clg.cases()[i]
    check_worlds(c.topo, c.blob, committed=True,
                 setup=lambda e: e.set_exclusive_levels(c.lv[1:], c.occ, level_n_domains=c.nd[1:]),
                 committed_levels=True)


# ---- errors, limits and handles

def raw_local(e, gb, n_alt, committed, assign):
    xh, p, nb, rounds = C.c_int32(-7), C.c_void_p(0), C.c_int64(-7), C.c_int32(9)
    i32 = _lib.i32p
    gbp = gb.ctypes.data_as(i32)
    ap = assign.ctypes.data_as(i32)
    if committed:
        rc = e.lib.rbgtopo_shard_place_groups_committed_ranked(e._h, gbp, len(gb), n_alt, ap, None, None,
                                                               C.byref(rounds), C.byref(xh), C.byref(p), C.byref(nb))
    else:
        rc = e.lib.rbgtopo_shard_place_groups_ranked(e._h, gbp, len(gb), n_alt, ap, None, None, C.byref(xh),
                                                     C.byref(p), C.byref(nb))
    return rc, xh.value, p.value, nb.value, rounds.value


def code(fn):
    try:
        fn()
    except RbgTopoError as e:
        return e.code
    return 0


def check_refused(topo, gb, expect=None, committed=False, n_alt=8, **kw):
    """The code of the world = 1 ranked call (expect, when given), on every rank of world 1 and 2, with nothing
    written: assign, the handle, the buffer and its size untouched, rounds 0."""
    e1 = TopoPlacer(device=0, **kw)
    e1.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    try:
        c1 = code(lambda: world1(e1, gb, n_alt, committed))
    finally:
        e1.close()
    assert c1 != 0 and (expect is None or c1 == expect), (c1, expect)
    expect = c1
    for W in (1, 2):
        engs = engines(topo, W, **kw)
        try:
            for e in engs:
                assign = np.full(max(int(gb[4]), 1), 12345, np.int32)
                rc, xh, p, nb, rounds = raw_local(e, gb, n_alt, committed, assign)
                assert rc == expect, (W, rc, expect)
                assert (assign == 12345).all() and xh == -7 and not p and nb == -7, (W, xh, p, nb)
                assert rounds == (0 if committed else 9)
        finally:
            close(engs)


def test_errors_are_those_of_world_1_with_nothing_written():
    case = gg.make_case(3, 33, exclusive=True)
    gb = case.blob
    for committed in (False, True):
        check_refused(case.topo, gb, EINVAL, committed, n_alt=9)
        check_refused(case.topo, gb, EINVAL, committed, n_alt=-1)
        for word, value in [(0, 0), (2, -1), (8 + 3, 0), (8 + 3, 17), (8 + 10, 1)]:
            b = gb.copy()
            b[word] = value
            check_refused(case.topo, b, None, committed)
    # a group at level 1 with levels installed, on a ctx without the level flag
    lv = gb.copy()
    lv[8 + 10] = 1
    levels = lo.random_levels(np.random.default_rng(1), case.topo.n, case.topo.domain, 1, [True])
    for committed in (False, True):
        e1 = TopoPlacer(device=0)
        e1.set_topology(case.topo.row_ptr, case.topo.col_idx, case.topo.edge_w, case.topo.free, case.topo.domain,
                        case.topo.domain_owner)
        e1.set_exclusive_levels(levels[1:], np.zeros((0, 3), np.int32))
        try:
            assert code(lambda: world1(e1, lv, 8, committed)) == ELIMIT
        finally:
            e1.close()
        engs = engines(case.topo, 2)
        try:
            for e in engs:
                e.set_exclusive_levels(levels[1:], np.zeros((0, 3), np.int32))
                rc = raw_local(e, lv, 8, committed, np.zeros(max(int(lv[4]), 1), np.int32))[0]
                assert rc == ELIMIT, rc
        finally:
            close(engs)


def test_exactness_bound_is_that_of_world_1():
    topo = synth.make_topology(256, seed=3, tiers=2, max_free=2)
    blob = lambda A: GroupsBuilder().add(Group(gid=1, roles=[(0, 40, 1, 0)], pair=[[1]], anchors=[(7, 0, A)],
                                               flags=0)).build()
    e1 = TopoPlacer(device=0)
    e1.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    try:
        lo_, hi = 1, 1 << 20   # the largest anchor count the ranked call accepts
        while hi - lo_ > 1:
            mid = (lo_ + hi) // 2
            if code(lambda: e1.place_groups_ranked(blob(mid), 0)) == 0:
                lo_ = mid
            else:
                hi = mid
        assert code(lambda: e1.place_groups_ranked(blob(lo_ + 1), 0)) == EINEXACT
    finally:
        e1.close()
    for committed in (False, True):
        check_refused(topo, blob(lo_ + 1), EINEXACT, committed, n_alt=0)
        check_worlds(topo, blob(lo_), n_alts=(8,), committed=committed, worlds=(2,))


def test_room_bitmap_limit_is_on_n():
    """N = 1 638 401 at world 2: ELIMIT, though each slab would fit; N = 1 638 400 is placed and ranked."""
    def topo_of(n):
        rp = (2 * np.arange(n + 1)).astype(np.int32)   # a ring: every node next to n - 1 and n + 1
        col = np.sort(np.stack([(np.arange(n) - 1) % n, (np.arange(n) + 1) % n], axis=1), axis=1).ravel().astype(np.int32)
        free = np.ones(n, np.int32)
        free[::7] = 2
        return synth.Topology(rp, col, np.ones(2 * n, np.int32), free, (np.arange(n) // 4096).astype(np.int32),
                              np.full((n + 4095) // 4096, -1, np.int32))
    b = GroupsBuilder()
    b.add(Group(gid=1, roles=[(0, 3, 1, 0), (1, 2, 2, 0)], pair=[[1, 1], [1, 1]], anchors=[(5, 0, 1)], flags=0))
    b.add(Group(gid=2, roles=[(0, 4, 1, 0)], pair=[[1]], anchors=[(1638399, 0, 2)], flags=0))
    gb = b.build()
    big = 200 * 1024 * 8
    check_refused(topo_of(big + 1), gb, ELIMIT)
    check_refused(topo_of(big + 1), gb, ELIMIT, committed=True)
    for committed in (False, True):
        check_worlds(topo_of(big), gb, n_alts=(8,), committed=committed, worlds=(2,))


def test_handles_refresh_reverse_order_release_and_double_merge():
    case = gg.make_case(6, 4097, scarce=True, exclusive=True)
    topo, gb = case.topo, case.blob
    e1 = TopoPlacer(device=0)
    e1.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    ref = e1.place_groups_ranked(gb, 8)
    cref = e1.place_groups_committed_ranked(gb, 8)
    groups, committed = e1.place_groups(gb), e1.place_groups_committed(gb)
    e1.close()
    engs = engines(topo, 2)
    try:
        R = int(gb[4])
        # two exchanges in flight on each ctx, merged in reverse order, with a refresh between the halves
        la = [e.shard_place_groups_ranked(gb, 8) for e in engs]
        lb = [e.shard_place_groups_committed_ranked(gb, 8) for e in engs]
        free2 = np.maximum(topo.free - 1, 0).astype(np.int32)
        for e in engs:
            e.update_nodes(free=free2)
        ka, kb = gather([(l[-2], l[-1]) for l in la]), gather([(l[-2], l[-1]) for l in lb])
        for e, l in zip(engs, lb):
            same((*l[:4], *e.shard_alternates_merge(l[-3], kb.data_ptr(), R, 8)), cref, "committed, second")
        for e, l in zip(engs, la):
            same((*l[:3], *e.shard_alternates_merge(l[-3], ka.data_ptr(), R, 8)), ref, "first")
            assert code(lambda: e.shard_alternates_merge(l[-3], ka.data_ptr(), R, 8)) == EINVAL   # consumed
        # a staged handle is not an exchange; null arguments leave the handle alive; release frees an unmerged one
        for e in engs:
            e.update_nodes(free=topo.free)
            h = e.stage_groups(gb)
            assert code(lambda: e.shard_alternates_merge(h, ka.data_ptr(), R, 8)) == EINVAL
            e.release(h)
            l = e.shard_place_groups_ranked(gb, 8)
            assert e.lib.rbgtopo_shard_alternates_merge(e._h, l[-3], None, None, None, None) == EINVAL
            e.release(l[-3])
            assert code(lambda: e.shard_alternates_merge(l[-3], ka.data_ptr(), R, 8)) == EINVAL
            assert code(lambda: e.release(l[-3])) == EINVAL
        # the other entry points on the same ctxs give what they gave before
        for e in engs:
            same(e.place_groups(gb), groups, "place_groups after exchanges")
            same(e.place_groups_committed(gb), committed, "committed after exchanges")
            assert code(lambda: e.place_groups_ranked(gb, 8)) == ELIMIT
            assert code(lambda: e.place_groups_committed_ranked(gb, 8)) == ELIMIT
        outs, _ = sharded(engs, gb, 8)
        for o in outs:
            same(o, ref, "again")
    finally:
        close(engs)


def test_high_level_methods_at_world_1_and_with_a_gather():
    case = gg.make_case(4, 130, scarce=True, exclusive=True)
    topo, gb = case.topo, case.blob
    e1 = TopoPlacer(device=0)
    e1.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    try:
        assert e1.places_sharded_ranked
        same(e1.place_groups_ranked_sharded(gb, 8), e1.place_groups_ranked(gb, 8), "world 1")
        same(e1.place_groups_committed_ranked_sharded(gb, 8), e1.place_groups_committed_ranked(gb, 8), "world 1")
        same(e1.place_groups_ranked_sharded(gb, 8, all_gather=lambda p, nb: gather([(p, nb)])),
             e1.place_groups_ranked(gb, 8), "world 1, gather")

        def failing(p, nb):
            raise OSError("collective failed")
        with pytest.raises(OSError):
            e1.place_groups_ranked_sharded(gb, 8, all_gather=failing)
        same(e1.place_groups_ranked_sharded(gb, 8), e1.place_groups_ranked(gb, 8), "after a failed gather")
    finally:
        e1.close()


WORKER = r'''
import os, sys
import numpy as np, torch, torch.distributed as dist
sys.path.insert(0, os.environ["RBG_ROOT"]); sys.path.insert(0, os.path.join(os.environ["RBG_ROOT"], "tests"))
import commit_gen as cg
import groups_gen as gg
from rbg_b200.engine import TopoPlacer
rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
def eng_of(topo, w, r):
    e = TopoPlacer(device=local, rank=r, world=w)
    e.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    return e
def bits(x):
    x = np.asarray(x)
    return x.view(np.uint32) if x.dtype == np.float32 else x
cases = [(gg.make_case(s, n, scarce=sc, exclusive=ex), False) for s, n, sc, ex in gg.CASES[:6]]
cases += [(c, True) for c in cg.cases()[::4]]
for case, committed in cases:
    e1, e = eng_of(case.topo, 1, 0), eng_of(case.topo, world, rank)
    for n_alt in (0, 8):
        if committed:
            ref, got = e1.place_groups_committed_ranked(case.blob, n_alt), e.place_groups_committed_ranked_sharded(case.blob, n_alt)
        else:
            ref, got = e1.place_groups_ranked(case.blob, n_alt), e.place_groups_ranked_sharded(case.blob, n_alt)
        for x, y in zip(got, ref):
            assert np.array_equal(bits(x), bits(y)), (rank, committed, n_alt)
    e1.close(); e.close()
dist.barrier()
if rank == 0: print("SHARD_ALTERNATES_OK", world)
dist.destroy_process_group()
'''


def test_plain_and_committed_over_nccl(tmp_path):
    import torch
    ngpu = torch.cuda.device_count()
    if ngpu < 2:
        # One GPU: NCCL needs one device per rank, so the same cases run with the ranks as contexts of this device
        # and a device copy as the all-gather (the tests above).
        test_generated_fleets(*gg.CASES[5])
        test_committed_batches(0)
        return
    world = 2 if ngpu < 4 else 4
    script = tmp_path / "shard_alternates_worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, RBG_ROOT=os.path.dirname(HERE))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
                        "--master-addr", "127.0.0.1", "--master-port", "29519", str(script)],
                       env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "SHARD_ALTERNATES_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
