"""GPU: rbgtopo_run_staged_chain on a caller stream, where it really chains.

The chain takes its programmatic form only when every handle runs on one stream, which without rbgtopo_set_stream never
happens (each batch has its own).  Every case here puts the context on a caller stream (kernel timing off, no library
switch) and queues a bounded sleep on that stream first: the whole chain is enqueued before the GPU reaches it, so the
passes run back to back and the dense-matrix kernel of pass k + 1 overlaps the selection kernel of pass k.  After the
chain every handle is compared bit for bit — assign, status, domain, every dense row (float32 bits) and top-K list a
pass defines (test_gpu_groups_limits.defined_rows) — with a plain run_staged of the same batch on an internal-stream
context, which is itself checked against the oracle's wave loop on the same raw GROUPS blob.  A correction of pass k landing after the re-emit of pass
k + n would show in the rows as a double correction even where the placements still look right."""
import os
import subprocess
import sys

import numpy as np
import pytest

import groups_gen as gg
from gpu_util import assert_same_result, new_engine, plan_result, sleep_on
from rbg_b200 import synth
from rbg_b200.blob import ROLE_EXCLUSIVE, Group, GroupsBuilder
from rbg_b200.engine import plan_steps
from test_gpu_groups_limits import check_handle, defined_rows, oracle_plan

pytestmark = pytest.mark.gpu


def _build(groups):
    gb = GroupsBuilder()
    for g in groups:
        gb.add(g)
    return gb.build()


def _tiny(gid):
    """One group, one role, one replica, no scheduled pod: k_plan_group's wave 0 waits and has nothing patched."""
    return Group(gid=gid, roles=[(0, 1, 1, ROLE_EXCLUSIVE)], pair=[[0]], anchors=[])


def _blobs(case, n, seed):
    """n distinct batches over one snapshot: the whole fleet (heavy, multi-wave groups that correct later waves), a
    one-role one-replica group, two groups, then random subsets of the fleet (1-3 groups when n is large)."""
    rng = np.random.default_rng(seed)
    gs = case.groups
    out = [_build(gs), _build([_tiny(9001)]), _build([_tiny(9002), gs[int(rng.integers(0, len(gs)))]])]
    while len(out) < n:
        k = int(rng.integers(1, 4)) if n > 8 else int(rng.integers(1, len(gs) + 1))
        pick = sorted(rng.choice(len(gs), size=min(k, len(gs)), replace=False).tolist())
        out.append(_build([gs[i] for i in pick]))
    return out[:n]


class Ref:
    """Plain passes on an internal-stream context: the expected result of every batch, checked against the oracle."""

    def __init__(self, topo, blobs, oracle=True, **kw):
        eng = new_engine(topo, **kw)
        self.want, self.sel = [], []   # sel: the replica rows and role rows a pass defines
        try:
            for gb in blobs:
                states, waves = oracle_plan(topo, gb)
                h = eng.stage_groups(gb)
                eng.run_staged(h, 1)
                if oracle:
                    check_handle(eng, topo, states, waves, gb, h)
                self.sel.append(defined_rows(topo, states, waves, gb))
                self.want.append(plan_result(eng, h, *self.sel[-1]))
                eng.release(h)
        finally:
            eng.close()

    def check(self, eng, hs, blobs, which, tag):
        for i in sorted(set(which)):
            assert_same_result(plan_result(eng, hs[i], *self.sel[i]), self.want[i], (tag, i))


def _on_caller_stream(eng):
    import torch
    st = torch.cuda.Stream()
    eng.set_stream(st.cuda_stream)
    return st


def chain_and_check(eng, st, ref, hs, blobs, counts, tag, order=None):
    """One chain per pass count over the batches `order` (default: all, in order), queued behind a sleep; then every
    batch the chain ran against the reference."""
    order = list(range(len(hs))) if order is None else order
    for passes in counts:
        sleep_on(st)
        eng.run_staged_chain([hs[i] for i in order], passes)
        ref.check(eng, hs, blobs, [order[k % len(order)] for k in range(passes)], (tag, passes))


@pytest.mark.parametrize("n", [2, 3, 4, 64])
def test_chain_on_a_caller_stream(n):
    """n = 2: every other pass reuses a batch's buffers, the tightest case for the transitive ordering of k_emit_rows'
    trailing griddepcontrol.wait; n = 64 is the ABI maximum.  Pass counts 1, n, 7n + 2 (ending mid-round) and 300."""
    case = gg.make_case(20 + n, 2049, n_groups=16)
    blobs = _blobs(case, n, n)
    ref = Ref(case.topo, blobs)
    eng = new_engine(case.topo)
    try:
        st = _on_caller_stream(eng)
        hs = [eng.stage_groups(gb) for gb in blobs]
        chain_and_check(eng, st, ref, hs, blobs, [1, n, 7 * n + 2, 300], ("n", n))
        if n == 2:   # tiny -> heavy as the first transition too
            chain_and_check(eng, st, ref, hs, blobs, [5], "reversed", order=[1, 0])
        for h in hs:
            eng.release(h)
    finally:
        eng.close()


@pytest.mark.parametrize("seed,n,scarce,excl,chunk", [(1, 7, False, True, 0), (4, 130, True, True, 0),
                                                      (5, 2049, False, True, 0), (9, 2049, False, False, 0),
                                                      (10, 1, False, True, 0), (6, 4097, True, True, 128)])
def test_chain_at_ragged_node_counts(seed, n, scarce, excl, chunk):
    """Ragged N (the tail mask of k_emit_rows), scarce capacity (status 1 / 2 groups), exclusive groups with fixed and
    preset domains (k_emit_rows<true>) and without (<false>), and 128-node chunks."""
    case = gg.make_case(seed, n, n_groups=12, scarce=scarce, exclusive=excl)
    blobs = _blobs(case, 3, seed)
    ref = Ref(case.topo, blobs, chunk_nodes=chunk)
    eng = new_engine(case.topo, chunk_nodes=chunk)
    try:
        st = _on_caller_stream(eng)
        hs = [eng.stage_groups(gb) for gb in blobs]
        chain_and_check(eng, st, ref, hs, blobs, [3, 23], ("N", n))
        for h in hs:
            eng.release(h)
    finally:
        eng.close()


def _placing_rows(topo, gb, exp):
    """Replica rows and role rows of the groups the oracle places completely (status 0): every wave of theirs is
    selected, so the rows a pass leaves for them are defined."""
    states, _ = oracle_plan(topo, gb)   # geometry only: the waves of each group
    rows, roles = [], []
    for stp in plan_steps(gb, topo.n, len(topo.domain_owner)):
        g, w = int(stp[0]), int(stp[1])
        if exp[g][1] == 0:
            wave = states[g].waves[w]
            rows += range(int(stp[4]), int(stp[4]) + sum(c for _, _, c in wave))
            roles += range(int(stp[5]), int(stp[5]) + len(wave))
    assert rows and roles
    return rows, roles


def _level_case(kind):
    """(topo, partitions, domains per level, GROUPS blob, occupancy records, level_placement flag).  "levels": a
    RBGTOPO_CFG_LEVEL_PLACEMENT context with groups at levels 0..3; "occupancy": a context without the flag whose
    level-0 groups see owners derived from the records (occupancy mode)."""
    import levels_oracle as lo
    from test_gpu_levels_place import fleet
    if kind == "levels":
        topo, lv, nd, gb, occ = fleet(44, 2049, "mixed", scarce=True)
        return topo, lv, nd, gb, occ, True
    case = gg.make_case(46, 2049, n_groups=12, scarce=True)
    topo, gb = case.topo, case.blob
    gids = [int(gb[8 + 12 * g]) for g in range(int(gb[2]))]
    lv = lo.random_levels(np.random.default_rng(46), topo.n, topo.domain, 3, [True, False, True])
    nd = [len(topo.domain_owner)] + [int(lv[L].max()) + 1 for L in range(1, lv.shape[0])]
    occ = lo.random_occ(np.random.default_rng(1046), topo.n, 3, gids[:4] + [999], topo.n // 6)
    return topo, lv, nd, gb, occ, False


def profile_chain(eng, st, hs, passes):
    """One chain of `passes` passes behind a sleep on the caller stream `st`, under torch.profiler (CUDA activities).
    Asserts that every k_emit_rows / k_plan_group of the call ran on the caller stream (the sleep's stream) and returns
    how many k_emit_rows of pass k + 1 started before k_plan_group of pass k ended.  Plain passes (the fallback) launch
    k_emit_rows in stream order behind the previous k_plan_group, so for them the count is 0; a chain overlaps as far
    as timing lets it."""
    import time

    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        # The profiler keeps only activities that start after its capture window opens, comparing GPU timestamps
        # converted to host time with the host clock.  That conversion has been seen off by more than the 50 ms of the
        # sleep (the sleep and the first passes were dropped behind a 10 ms margin), so the margin on the host is half
        # a second.
        time.sleep(0.5)
        sleep_on(st)
        eng.run_staged_chain(hs, passes)
        torch.cuda.synchronize()
    kern = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    sleeps = [e for e in kern if "spin_kernel" in e.name or "sleep" in e.name.lower()]   # torch.cuda._sleep
    emit = sorted((e for e in kern if "k_emit_rows" in e.name), key=lambda e: e.time_range.start)
    plan = sorted((e for e in kern if "k_plan_group" in e.name), key=lambda e: e.time_range.start)
    assert len(sleeps) == 1 and len(emit) == passes and len(plan) == passes, (len(sleeps), len(emit), len(plan))
    streams = {e.device_resource_id for e in emit + plan}
    assert streams == {sleeps[0].device_resource_id}, (streams, sleeps[0].device_resource_id)
    return sum(1 for k in range(passes - 1) if emit[k + 1].time_range.start < plan[k].time_range.end)


@pytest.mark.parametrize("kind", ["levels", "occupancy"])
def test_chain_at_exclusive_levels_and_in_occupancy_mode(kind):
    """The same batch staged twice chains through two handles, on a level-placement context with groups at levels
    0..3 and on an occupancy-mode context with level-0 groups: placements against the oracle on each group's level
    view, rows and lists against plain passes.  A profiled chain shows that the chained form ran, not the fallback."""
    import levels_oracle as lo
    import levels_view as lvw
    from test_gpu_levels_place import assert_fleet
    from rbg_b200.engine import TopoPlacer
    topo, lv, nd, gb, occ, flag = _level_case(kind)
    exp, _ = lvw.expected_fleet(topo, lv, lo.derive_level_owner(lv, occ), nd, gb)
    rows, roles = _placing_rows(topo, gb, exp)

    def engine():
        e = TopoPlacer(device=0, level_placement=flag)
        e.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
        e.set_exclusive_levels(lv[1:], occ, level_n_domains=nd[1:])
        return e
    r = engine()
    try:
        h = r.stage_groups(gb)
        r.run_staged(h, 1)
        want = plan_result(r, h, rows, roles)
        assert_fleet(want[:3], exp, gb, "plain", staged=True)
    finally:
        r.close()
    eng = engine()
    try:
        st = _on_caller_stream(eng)
        hs = [eng.stage_groups(gb), eng.stage_groups(gb)]
        for passes in (2, 16, 41):
            sleep_on(st)
            eng.run_staged_chain(hs, passes)
            for h in hs[:min(passes, 2)]:
                got = plan_result(eng, h, rows, roles)
                assert_fleet(got[:3], exp, gb, ("chain", passes), staged=True)
                assert_same_result(got, want, (kind, passes))
        if not (os.environ.get("RBGTOPO_NO_PDL") or os.environ.get("RBGTOPO_CONCURRENT_PLAN")):   # those never chain
            overlap = profile_chain(eng, st, hs, 20)
            print(f"\n[chain witness] {kind}: {overlap} of 19 k_emit_rows started before the previous k_plan_group ended")
            assert overlap > 0, "plain passes ran: the level batches did not chain"
        for h in hs:
            got = plan_result(eng, h, rows, roles)
            assert_same_result(got, want, (kind, "profiled"))
    finally:
        eng.close()


@pytest.mark.parametrize("world", [2, 4])
def test_chain_per_rank_on_one_device(world):
    """world = 2 and 4 contexts of one device (replicated selection, a column slab of the dense matrix each): every rank
    chains on its own caller stream, then all ranks on one caller stream.  Each rank's slab against world = 1."""
    import torch
    from rbg_b200.engine import TopoPlacer
    case = gg.make_case(31, 4097, n_groups=12)
    blobs = _blobs(case, 3, 31)
    ref = Ref(case.topo, blobs)
    topo = case.topo
    engs = []
    try:
        for r in range(world):
            e = TopoPlacer(device=0, rank=r, world=world)
            e.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
            engs.append(e)
        hss = [[e.stage_groups(gb) for gb in blobs] for e in engs]

        def check(passes, tag):
            for r, (e, hs) in enumerate(zip(engs, hss)):
                lo, hi = e.slab()
                for i in sorted(set(k % 3 for k in range(passes))):
                    a, s, d, rows, topk = ref.want[i]
                    assert_same_result(plan_result(e, hs[i], *ref.sel[i]), (a, s, d, rows[:, lo:hi], topk),
                                       (tag, world, r, i))
        streams = [torch.cuda.Stream() for _ in engs]
        for e, st in zip(engs, streams):
            e.set_stream(st.cuda_stream)
            sleep_on(st)
        for e, hs in zip(engs, hss):
            e.run_staged_chain(hs, 23)
        check(23, "own streams")
        one = torch.cuda.Stream()
        for e in engs:
            e.set_stream(one.cuda_stream)
        sleep_on(one)
        for e, hs in zip(engs, hss):
            e.run_staged_chain(hs, 7)
        check(7, "one stream")
    finally:
        for e in engs:
            e.close()


def _beyond_smem_group(rng, n):
    """A 16-role group with scheduled pods on 120 distinct nodes: its table does not fit k_plan_group's shared memory
    (test_gpu_groups_limits.test_tables_beyond_shared_memory_take_the_per_wave_path)."""
    from test_gpu_groups_limits import _wide_group
    wide = _wide_group(rng, 16, 5, n)
    p = np.asarray(wide.pair)
    p[:, 15] = 0
    wide.pair = p.tolist()
    nodes = rng.choice(n, size=120, replace=False)
    wide.anchors = [(int(x), 15, 1) for x in nodes] + [(int(x), int(rng.integers(0, 15)), 2) for x in nodes[:12]]
    return wide


def test_chain_fallbacks_give_the_same_bits():
    """The documented fallbacks to plain passes: a batch whose table exceeds shared memory in the chain, and kernel
    timing turned on (and off again) between chains still queued behind the sleep."""
    n = 4097
    topo = synth.make_topology(n, seed=3, tiers=4, max_free=4)
    rng = np.random.default_rng(120)
    from test_gpu_groups_limits import _one_role_groups
    small = _one_role_groups(rng, 12, 10, n)
    blobs = [_build(small[:6]), _build([_beyond_smem_group(rng, n)] + small[6:]), _build(small[6:9])]
    ref = Ref(topo, blobs)
    eng = new_engine(topo)
    try:
        st = _on_caller_stream(eng)
        hs = [eng.stage_groups(gb) for gb in blobs]
        chain_and_check(eng, st, ref, hs, blobs, [3, 11], "beyond shared memory")
        sleep_on(st)
        eng.run_staged_chain([hs[0], hs[2]], 9)
        eng.set_kernel_timing(True)
        eng.run_staged_chain([hs[2], hs[0]], 6)
        eng.set_kernel_timing(False)
        eng.run_staged_chain([hs[0], hs[2]], 5)
        ref.check(eng, hs, blobs, [0, 2], "timing toggled")
        for h in hs:
            eng.release(h)
    finally:
        eng.close()


def bench_fleet():
    """bench.py's cfg3: (topology, fleet specs, GROUPS blob of 1 024 mooncake groups x 10 000 nodes, (replica rows, role
    rows)): every group places everything, so every row is defined."""
    import bench
    from rbg_b200.plugin import B200TopoPodGroupManager
    n, groups = 10000, 1024
    topo = synth.make_topology(n, seed=0, tiers=4, samples_per_tier=5)
    specs = bench.fleet_spec("mooncake", groups, n)
    gblob, _ = B200TopoPodGroupManager(None).groups_blob(bench.to_plugin(specs))
    P = sum(len(gg.waves_of([tuple(int(v) for v in gblob[o:o + 4])
                             for o in range(int(gblob[8 + 12 * g + 4]), int(gblob[8 + 12 * g + 4]) + 4 * int(gblob[8 + 12 * g + 3]), 4)]))
            for g in range(groups))
    return topo, specs, gblob, (range(int(gblob[4])), range(P))


def test_bench_shape_chain():
    """What bench.py --slots 4 times: 4 staged copies of the mooncake fleet (1 024 groups x 10 000 nodes), 50 chained
    passes.  Each copy against plain passes bit for bit and against the oracle on 128 sampled groups."""
    import bench
    n, groups = 10000, 1024
    topo, specs, gblob, sel = bench_fleet()
    eng = new_engine(topo)
    try:
        h = eng.stage_groups(gblob)
        eng.run_staged(h, 1)
        want = plan_result(eng, h, *sel)
        eng.release(h)
        st = _on_caller_stream(eng)
        hs = [eng.stage_groups(gblob) for _ in range(4)]
        sleep_on(st)
        eng.run_staged_chain(hs, 50)
        sample = sorted(set(int(i) for i in np.linspace(0, groups - 1, 128)))
        for k, h in enumerate(hs):
            got = plan_result(eng, h, *sel)
            assert_same_result(got, want, ("copy", k))
            par = bench.parity_check(eng, topo, specs, gblob, h, got[:3], sample, 0, n, 8)
            assert par["ok"] and par["rows_checked"] == 128 * 7 and par["waves"] == 3, (k, par)
        for h in hs:
            eng.release(h)
    finally:
        eng.close()


def test_chain_runs_on_the_caller_stream_under_the_profiler():
    """Witness that the chain ran as one: with torch.profiler around one chain of the n = 4 case, every k_emit_rows /
    k_plan_group of the call ran on the caller stream (the stream of the sleep queued on it).  Prints how many
    k_emit_rows of pass k + 1 started before k_plan_group of pass k ended (timing-dependent: reported, not asserted)."""
    import torch
    case = gg.make_case(24, 2049, n_groups=16)
    blobs = _blobs(case, 4, 4)
    ref = Ref(case.topo, blobs, oracle=False)
    eng = new_engine(case.topo)
    try:
        st = _on_caller_stream(eng)
        hs = [eng.stage_groups(gb) for gb in blobs]
        sleep_on(st, 1000)    # warm-up: modules loaded, buffers touched
        eng.run_staged_chain(hs, 4)
        torch.cuda.synchronize()
        passes = 40
        overlap = profile_chain(eng, st, hs, passes)
        print(f"\n[chain witness] n = 4, {passes} passes: {overlap} of {passes - 1} k_emit_rows started before the "
              f"previous pass's k_plan_group ended")
        ref.check(eng, hs, blobs, range(4), "profiled")
        for h in hs:
            eng.release(h)
    finally:
        eng.close()


@pytest.mark.parametrize("var", ["RBGTOPO_NO_PDL", "RBGTOPO_CONCURRENT_PLAN"])
def test_chain_variants_in_a_subprocess(var):
    """RBGTOPO_NO_PDL: plain stream order instead of the programmatic chain; RBGTOPO_CONCURRENT_PLAN: k_plan_group on the
    second stream beside the dense-matrix kernel (no chain).  The library reads them when it loads."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ)
    env[var] = "1"
    r = subprocess.run(
        [sys.executable, "-m", "pytest", "tests/test_gpu_chain.py", "-q", "-m", "gpu", "-x",
         "-k", "test_chain_on_a_caller_stream or ragged or levels or fallbacks"],
        cwd=root, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert "passed" in r.stdout
