"""GPU, ONE device: the all-gather selection scheme on node-axis shards at its limits, and the same pipeline with the
exchange done inside the library (rbgtopo_run_staged_p2p, p2p.cuh).  Every rank is a context on the same GPU.  The host
all-gather concatenates the ranks' key buffers with a device copy (test_gpu_shard_single); the p2p form stores every
list into every rank's exchange buffer and acquire-waits on release flags.

The designed cases come from tests/allgather_limits_cases.py (checked on the CPU by test_allgather_limits_cases.py):
merges over 3 to 16 slabs, exclusive steps without a fixed domain, multi-wave plans chained through the plan blob, a
hub-anchored batch past the fast table, steps and plans at exclusive levels 4 to 7.  Every output on every rank is
compared bit for bit with the CPU oracle: placements, status and domain, this rank's slab of every dense row, every
merged list.  The file also runs the exchange buffer at its edges (a wave of exactly rows_cap role rows at both
parities, rows_cap + 1 rows before and in the middle of a pass, rows_cap = 1, re-export, iters = 4, 32 waves of one
and two phases), checks the peer-byte count, and enqueues two handles back to back on every rank.

On one device the ranks' spinning consumers must leave SMs for their producers: every pass here keeps each wave at
<= 64 steps for world >= 8, and the consumer CTAs of all ranks under a quarter of what the device holds.  They must
also leave the device's hardware queues to the producers.  A process feeds its streams to the device through
CUDA_DEVICE_MAX_CONNECTIONS queues (8 by default), assigned round-robin in creation order.  When two ranks' batch
streams land on one queue, a consumer spinning at its head keeps the other rank's producer from starting until the
bounded wait times out; which streams share a queue depends on every stream the process created before.  Ranks on GPUs
of their own share no queue.  So every test here runs in a fresh process with 32 queues, where the batch streams of up
to 16 ranks, created one after another, each get a queue of their own.  And a process loads a kernel's module when
it first launches it, which waits for the kernels running on the device: a producer launched for the first time while
another rank's consumer spins never starts.  Every p2p pass here follows a host all-gather pass of the same batch on the
same contexts, which loads every kernel the pass launches."""
import json
import os
import subprocess
import sys
import time

import numpy as np
import pytest

import allgather_limits_cases as C
import levels_limits_cases as LC
import levels_oracle as lo
import steps_gen as sg
from oracle import placer as oracle_placer
from rbg_b200 import synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, STEP_GANG, BlobBuilder, Group, GroupsBuilder, Step
from rbg_b200.engine import RbgTopoError, plan_steps
from test_gpu_levels_limits import install, view_step
from test_gpu_levels_place import assert_fleet, engine
from test_gpu_shard_single import _engines, _gather
from test_gpu_steps_limits import _all_gather, _check_rank, _heavy_batch

pytestmark = pytest.mark.gpu

ELIMIT = -6
SMALL_CAP = 512


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _in_child(fn, *args):
    """fn(*args) of this module in a fresh process with 32 hardware queues (module docstring)."""
    code = ("import json, sys; sys.path[:0] = [sys.argv[1], sys.argv[1] + '/tests']; "
            "import test_gpu_allgather_limits as t; getattr(t, sys.argv[2])(*json.loads(sys.argv[3])); print('child OK')")
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32")
    r = subprocess.run([sys.executable, "-c", code, ROOT, fn, json.dumps(list(args))], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "child OK" in r.stdout, r.stdout[-3000:] + r.stderr[-4000:]


def _warm_up(engs, blob, groups=False):
    """A host all-gather pass of the batch on every rank, results unchecked: it loads every kernel a p2p pass of the
    batch launches (module docstring)."""
    hs = [e.stage_groups(blob) if groups else e.stage(blob) for e in engs]
    try:
        for w in range(engs[0].shard_waves(hs[0]) if groups else 1):
            allk = _gather([e.shard_wave_score(h, w) for e, h in zip(engs, hs)])
            m = [e.shard_wave_merge(h, w, allk.data_ptr()) for e, h in zip(engs, hs)]
            all2 = _gather([(x[1], x[2]) for x in m]) if m[0][0] else None
            for e, h in zip(engs, hs):
                e.shard_wave_assign(h, w, all2.data_ptr() if all2 is not None else None)
        import torch
        torch.cuda.synchronize()
    finally:
        for e, h in zip(engs, hs):
            e.release(h)


def _code(fn, *args):
    with pytest.raises(RbgTopoError) as ei:
        fn(*args)
    return ei.value.code


def _room(world, steps_per_wave):
    """Each wave's consumer CTAs over all ranks (k_merge / k_greedy: 4 steps per CTA) stay under a quarter of the
    CTAs the device holds (16 per SM)."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for n in steps_per_wave:
        assert world < 8 or n <= 64, (world, n)
        assert world * -(-n // 4) < sms * 16 // 4, (world, n, sms)


def _connect(engs, rows_cap=SMALL_CAP):
    ptrs = [e.p2p_export(rows_cap=rows_cap)[1] for e in engs]
    for e in engs:
        e.p2p_import(ptrs=ptrs)


def _close(engs):
    for e in engs:
        e.close()


def _p2p_steps(engs, topo, blob, ref, tag, iters=1):
    """run_staged_p2p on every rank, every output checked, no timeout, the peer-byte count of one pass."""
    import torch
    world = len(engs)
    hs = [e.stage(blob) for e in engs]
    try:
        for e, h in zip(engs, hs):
            e.run_staged_p2p(h, iters)
        torch.cuda.synchronize()
        want = C.peer_bytes("steps", blob, topo, world)
        for r, (e, h) in enumerate(zip(engs, hs)):
            st = e.p2p_stats()
            assert not st["timed_out"] and st["peer_bytes_last_pass"] == want, tag + (r, st, want)
            _check_rank(e, h, ref, tag + ("p2p", r))
    finally:
        for e, h in zip(engs, hs):
            e.release(h)


# ---------------------------------------------------------------- designed step batches
@pytest.mark.parametrize("family", ["merge", "excl"])
def test_step_cases(family):
    """Every designed step case of the family at every world it names: host all-gather, then p2p."""
    _in_child("_step_family", family)


def _step_family(family):
    for fam, name in C.all_step_cases():
        if fam == family:
            _step_case(fam, name)


def _step_case(family, name):
    topo, blob, info = C.step_case(family, name)
    ref = oracle_placer.place(topo, blob)
    C.step_pre(family, name, topo, blob, info, ref)
    for world in info["worlds"]:
        _room(world, [int(blob[2])])
        engs = _engines(topo, world)
        try:
            _connect(engs)
            _all_gather(engs, blob, ref, (name, world))
            _p2p_steps(engs, topo, blob, ref, (name, world))
        finally:
            _close(engs)


# ---------------------------------------------------------------- designed plans
def _check_plan(e, h, topo, gblob, states, waves, tag):
    """This rank's slab of every row every wave the oracle ran defines, every merged list, every group's result."""
    from test_gpu_groups_limits import group_slices
    a, s, d = e.fetch(h)
    lo_, hi = e.slab()
    first = {(int(st[0]), int(st[1])): (int(st[4]), int(st[5])) for st in plan_steps(gblob, topo.n, len(topo.domain_owner))}
    lost = set()
    for w, gis, _, r in waves:
        off = rr = 0
        for gi in gis:
            wave = states[gi].waves[w]
            cnt, P = sum(c for _, _, c in wave), len(wave)
            if gi not in lost:
                row0, role0 = first[(gi, w)]
                for j in range(cnt):
                    got = e.read_scores(h, row0 + j)
                    assert np.array_equal(got.view(np.uint32), r["matrix"][off + j, lo_:hi].view(np.uint32)), tag + ("row", w, gi, j)
                for p in range(P):
                    assert np.array_equal(e.read_topk(h, role0 + p, 32), r["topk"][rr + p]), tag + ("topk", w, gi, p)
                if (r["assign"][off:off + cnt] < 0).any():
                    lost.add(gi)
            off += cnt
            rr += P
    for i, (st, sl) in enumerate(zip(states, group_slices(states))):
        res = st.result()
        if res["status"] == 1:
            assert int(s[i]) == 1, tag + (i,)
            continue
        assert a[sl].tolist() == st.assign_in_group_order(), tag + (i,)
        assert (int(s[i]), int(d[i])) == (res["status"], res["domain"]), tag + (i,)


def _wave_sizes(topo, gblob):
    ps = plan_steps(gblob, topo.n, len(topo.domain_owner))
    return np.bincount(ps[:, 1]).tolist()


def _plan_both(engs, topo, gblob, plan, tag):
    import torch
    states, waves = plan
    world = len(engs)
    _room(world, _wave_sizes(topo, gblob))
    hs = [e.stage_groups(gblob) for e in engs]
    try:
        for w in range(engs[0].shard_waves(hs[0])):
            allk = _gather([e.shard_wave_score(h, w) for e, h in zip(engs, hs)])
            m = [e.shard_wave_merge(h, w, allk.data_ptr()) for e, h in zip(engs, hs)]
            all2 = _gather([(x[1], x[2]) for x in m]) if m[0][0] else None
            for e, h in zip(engs, hs):
                e.shard_wave_assign(h, w, all2.data_ptr() if all2 is not None else None)
        for r, (e, h) in enumerate(zip(engs, hs)):
            _check_plan(e, h, topo, gblob, states, waves, tag + ("all-gather", r))
    finally:
        for e, h in zip(engs, hs):
            e.release(h)
    hs = [e.stage_groups(gblob) for e in engs]
    try:
        for e, h in zip(engs, hs):
            e.run_staged_p2p(h, 1)
        torch.cuda.synchronize()
        want = C.peer_bytes("plan", gblob, topo, world)
        for r, (e, h) in enumerate(zip(engs, hs)):
            st = e.p2p_stats()
            assert not st["timed_out"] and st["peer_bytes_last_pass"] == want, tag + (r, st, want)
            _check_plan(e, h, topo, gblob, states, waves, tag + ("p2p", r))
    finally:
        for e, h in zip(engs, hs):
            e.release(h)


@pytest.mark.parametrize("name", C.PLAN_CASES)
def test_plan_cases(name):
    _in_child("_plan_case", name)


def _plan_case(name):
    topo, gblob, info = C.plan_case(name)
    plan = C.plan_pre(name, topo, gblob, info)
    for world in info["worlds"]:
        engs = _engines(topo, world)
        try:
            _connect(engs)
            _plan_both(engs, topo, gblob, plan, (name, world))
        finally:
            _close(engs)


# ---------------------------------------------------------------- the global candidate list at world 8
def test_global_candidate_list_at_world_8():
    _in_child("_global_candidate_list")


def _global_candidate_list():
    case = sg.make_case(22, 2049, 17)
    topo = case.topo
    ref = oracle_placer.place(topo, case.blob)
    heavy = sg.build(_heavy_batch(topo, 22))
    href = oracle_placer.place(topo, heavy)
    assert ref["rc"] == 0 and href["rc"] == 0
    engs = _engines(topo, 8)
    try:
        _connect(engs)
        _all_gather(engs, heavy, href, ("heavy", 8))                  # shard_score takes k_select
        hs = [e.stage(heavy) for e in engs]
        try:
            for r, (e, h) in enumerate(zip(engs, hs)):
                assert _code(e.run_staged_p2p, h, 1) == ELIMIT, r
        finally:
            for e, h in zip(engs, hs):
                e.release(h)
        _p2p_steps(engs, topo, case.blob, ref, ("after ELIMIT", 8))
    finally:
        _close(engs)


# ---------------------------------------------------------------- exclusive levels 4..7 through p2p
@pytest.mark.parametrize("k", [0, 1])
def test_levels_through_p2p(k):
    _in_child("_levels_through_p2p", k)


def _levels_through_p2p(k):
    """Steps and a plan at keys 4..7 with owners derived from occupancy records, through run_staged_p2p at world 4."""
    import torch
    world = 4
    c = LC.keys47(*LC.KEYS47[k])
    owner = lo.derive_level_owner_fast(c.lv, c.occ)
    steps = LC.steps47(c, world)[:-1]
    assert {st.level for st in steps} >= {6, 7}
    refs = [view_step(c, owner, st) for st in steps]
    bb = BlobBuilder()
    for st in steps:
        bb.add(st)
    blob = bb.build()
    import levels_view as lvw
    exp_fleet, _ = lvw.expected_fleet(c.topo, c.lv, owner, c.nd, c.gblob)
    engs = [engine(c.topo, rank=r, world=world) for r in range(world)]
    try:
        for e in engs:
            install(e, c)
        _connect(engs)
        _warm_up(engs, blob)
        _warm_up(engs, c.gblob, groups=True)
        hs = [e.stage(blob) for e in engs]
        for e, h in zip(engs, hs):
            e.run_staged_p2p(h, 1)
        torch.cuda.synchronize()
        for r, (e, h) in enumerate(zip(engs, hs)):
            assert not e.p2p_stats()["timed_out"]
            a, s, d = e.fetch(h)
            off = 0
            lo_, hi = e.slab()
            for i, (st, ref) in enumerate(zip(steps, refs)):
                R = st.n_replicas
                rd = ref["domain"][0] // 2 if ref["domain"][0] >= 0 else -1
                assert a[off:off + R].tolist() == ref["assign"].tolist() and int(s[i]) == int(ref["status"][0]), (r, i)
                assert int(d[i]) == rd, (r, i)
                for j in range(R):
                    got = e.read_scores(h, off + j)
                    assert np.array_equal(got.view(np.uint32), ref["matrix"][j, lo_:hi].view(np.uint32)), (r, i, j)
                off += R
            e.release(h)
        hs = [e.stage_groups(c.gblob) for e in engs]
        for e, h in zip(engs, hs):
            e.run_staged_p2p(h, 1)
        torch.cuda.synchronize()
        for r, (e, h) in enumerate(zip(engs, hs)):
            assert not e.p2p_stats()["timed_out"]
            assert_fleet(e.fetch(h), exp_fleet, c.gblob, f"p2p rank {r}", staged=True)
            e.release(h)
    finally:
        _close(engs)


# ---------------------------------------------------------------- the exchange buffer at its edges
def _rows_blob(topo, rows, seed):
    """Steps of up to 8 one-replica roles, `rows` role rows in all."""
    rng = np.random.default_rng(seed)
    bb = BlobBuilder()
    gid = 0
    while rows > 0:
        P = min(8, rows)
        bb.add(Step(gid=gid, roles=[(1, int(rng.integers(0, 2)), int(rng.integers(1, 4)), 0) for _ in range(P)],
                       pair=np.eye(P, dtype=int).tolist(),
                       anchors=[(int(rng.integers(0, topo.n)), 0, 1)]))
        rows -= P
        gid += 1
    return bb.build()


def _wide_plan(groups, waves_at_level1):
    """Groups of one one-replica role at level 0 and `waves_at_level1` roles of one replica at level 1: wave 0 has one
    role row per group, wave 1 that many per group."""
    gb = GroupsBuilder()
    for g in range(groups):
        roles = [(0, 1, 1, 0)] + [(1, 1, 1, 0)] * waves_at_level1
        q = len(roles)
        gb.add(Group(gid=g, roles=roles, pair=np.eye(q, dtype=int).tolist()))
    return gb.build()


def test_exchange_buffer_edges_at_world_16():
    _in_child("_exchange_buffer_edges")


def _exchange_buffer_edges():
    import torch
    world, cap = 16, 64
    topo = synth.make_topology(2049, seed=5, tiers=3)
    exact = _rows_blob(topo, cap, 1)
    over = _rows_blob(topo, cap + 1, 2)
    assert int(exact[5]) == cap and int(over[5]) == cap + 1
    ref = oracle_placer.place(topo, exact)
    assert ref["rc"] == 0
    engs = _engines(topo, world)
    try:
        _connect(engs, cap)
        _warm_up(engs, exact)
        _warm_up(engs, _wide_plan(9, 8), groups=True)
        # exactly rows_cap rows: pass 1 uses parity 1, whose last source slot ends where the flag block starts; pass 2
        # parity 0
        for rep in range(2):
            _p2p_steps(engs, topo, exact, ref, ("exact", rep))
        hs = [e.stage(over) for e in engs]
        try:
            for r, (e, h) in enumerate(zip(engs, hs)):
                assert _code(e.run_staged_p2p, h, 1) == ELIMIT, r
        finally:
            for e, h in zip(engs, hs):
                e.release(h)
        # a plan whose wave 0 fits (9 rows) and whose wave 1 does not (72): refused in the middle of the pass on
        # every rank, after wave 0 was enqueued; the next pass still lines up across the ranks
        mid = _wide_plan(9, 8)
        assert _wave_sizes(topo, mid) == [9, 9]
        hs = [e.stage_groups(mid) for e in engs]
        try:
            for r, (e, h) in enumerate(zip(engs, hs)):
                assert _code(e.run_staged_p2p, h, 1) == ELIMIT, r
        finally:
            for e, h in zip(engs, hs):
                e.release(h)
        torch.cuda.synchronize()
        _p2p_steps(engs, topo, exact, ref, ("after mid-pass ELIMIT",))
        # re-export with another rows_cap, re-import, run again; then iters = 4 in one call
        _connect(engs, 2 * cap)
        _p2p_steps(engs, topo, over, oracle_placer.place(topo, over), ("re-exported",))
        _p2p_steps(engs, topo, exact, ref, ("iters 4",), iters=4)
    finally:
        _close(engs)


def test_rows_cap_one_and_world_17():
    _in_child("_rows_cap_one_and_world_17")


def _rows_cap_one_and_world_17():
    topo = synth.make_topology(1000, seed=3, tiers=2)
    blob = _rows_blob(topo, 1, 3)
    ref = oracle_placer.place(topo, blob)
    engs = _engines(topo, 3)
    try:
        _connect(engs, 1)
        _warm_up(engs, blob)
        _p2p_steps(engs, topo, blob, ref, ("rows_cap 1",))
    finally:
        _close(engs)
    engs = _engines(topo, 17)
    try:
        assert _code(engs[0].p2p_export, 8) == ELIMIT
    finally:
        _close(engs)


def _long_plan(n, plain_levels, plain_pending, excl_levels):
    """A plain group of `plain_levels` levels of `plain_pending` replicas each (ceil(pending / 32) waves per level), an
    exclusive group of `excl_levels` one-replica levels and an exclusive gang group of two-wave levels: the exclusive
    waves (two phases) come first, then the plain ones (one phase)."""
    gb = GroupsBuilder()
    gb.add(Group(gid=1, roles=[(lv, plain_pending, 1, 0) for lv in range(plain_levels)],
                 pair=np.eye(plain_levels, dtype=int).tolist()))
    gb.add(Group(gid=2, roles=[(lv, 1, 1, ROLE_EXCLUSIVE) for lv in range(excl_levels)],
                 pair=np.ones((excl_levels, excl_levels), int).tolist(), flags=STEP_EXCLUSIVE))
    gb.add(Group(gid=3, roles=[(lv, 33, 1, ROLE_EXCLUSIVE if lv % 2 else 0) for lv in range(5)],
                 pair=np.eye(5, dtype=int).tolist(), flags=STEP_EXCLUSIVE | STEP_GANG))
    return gb.build()


def _domain_topo(n, seed):
    rng = np.random.default_rng(seed)
    free = rng.integers(3, 6, n).astype(np.int32)
    return C.snapshot(n, free, (np.arange(n) // 1024).astype(np.int32))


def test_32_waves_of_one_and_two_phases():
    _in_child("_32_waves")


def _32_waves():
    """A plan of 32 waves: the exclusive groups' waves take two phases, the plain group's later ones one.  (More waves
    need a plain group of more replicas, whose last steps carry more patched nodes than k_shard_select's table holds on
    the sharded path: at about 100 and at 48 waves the pass is refused with RBGTOPO_ELIMIT.)"""
    import torch
    world = 4
    topo = _domain_topo(4096, 11)
    gblob = _long_plan(topo.n, 16, 33, 13)
    ph = C.phases_rows("plan", gblob, topo)
    assert len(ph) == 32 and {p for p, _ in ph} == {1, 2}
    states, waves = C.oracle_plan(topo, gblob)
    engs = _engines(topo, world)
    try:
        _connect(engs)
        _plan_both(engs, topo, gblob, (states, waves), ("32 waves",))
        # the same plan twice in one call
        hs = [e.stage_groups(gblob) for e in engs]
        try:
            for e, h in zip(engs, hs):
                e.run_staged_p2p(h, 2)
            torch.cuda.synchronize()
            for r, (e, h) in enumerate(zip(engs, hs)):
                assert not e.p2p_stats()["timed_out"]
                assert e.p2p_stats()["peer_bytes_last_pass"] == C.peer_bytes("plan", gblob, topo, world)
                _check_plan(e, h, topo, gblob, states, waves, ("32 waves, iters 2", r))
        finally:
            for e, h in zip(engs, hs):
                e.release(h)
    finally:
        _close(engs)


# ---------------------------------------------------------------- several handles in flight
def _in_flight(profiled):
    """Every rank enqueues a long plan h1 and at once a short batch h2 (each handle has a stream of its own), with no
    synchronisation in between.  Both must match the oracle with no timed-out wait.  profiled: under torch.profiler the
    passes must also be ordered on the device: the ranks' h2 passes can be paired with their h1 passes so that each h2's
    first k_shard_select starts after its h1's last k_greedy ended (sorted starts dominate sorted ends), which holds when
    every rank's h2 waits for its h1."""
    import contextlib

    import torch
    from torch.profiler import ProfilerActivity, profile
    from test_gpu_parity import _random_steps
    world = 4
    topo = _domain_topo(4096, 12)
    gblob = _long_plan(topo.n, 8, 64, 9)
    states, waves = C.oracle_plan(topo, gblob)
    blob = _random_steps(topo, 77, 12, excl=False, gang=True)
    ref = oracle_placer.place(topo, blob)
    assert ref["rc"] == 0
    n_waves = len(C.phases_rows("plan", gblob, topo))
    assert n_waves >= 16
    _room(world, [a + int(blob[2]) for a in _wave_sizes(topo, gblob)])   # both passes' consumers at once, were they to overlap
    engs = _engines(topo, world)
    try:
        _connect(engs)
        _warm_up(engs, gblob, groups=True)
        _warm_up(engs, blob)
        h1 = [e.stage_groups(gblob) for e in engs]
        h2 = [e.stage(blob) for e in engs]
        torch.cuda.synchronize()
        with (profile(activities=[ProfilerActivity.CUDA]) if profiled else contextlib.nullcontext()) as prof:
            time.sleep(0.5)     # activities that start before the capture window opens are dropped (test_gpu_chain)
            for e, h in zip(engs, h1):
                e.run_staged_p2p(h, 1)
            for e, h in zip(engs, h2):
                e.run_staged_p2p(h, 1)
            torch.cuda.synchronize()
        for r, e in enumerate(engs):
            assert not e.p2p_stats()["timed_out"], r
            _check_plan(e, h1[r], topo, gblob, states, waves, ("in flight h1", r))
            _check_rank(e, h2[r], ref, ("in flight h2", r))
        if not profiled:
            return
        kern = [k for k in prof.events() if k.device_type == torch.autograd.DeviceType.CUDA]
        by_stream = {}
        for k in kern:
            if "k_shard_select" in k.name or "k_greedy" in k.name:
                by_stream.setdefault(k.device_resource_id, []).append(k)
        greedy = {s: sum(1 for k in ks if "k_greedy" in k.name) for s, ks in by_stream.items()}
        long_ = [s for s, g in greedy.items() if g == n_waves]
        short = [s for s, g in greedy.items() if g == 1]
        assert len(long_) == world and len(short) == world, greedy
        ends = sorted(max(k.time_range.end for k in by_stream[s] if "k_greedy" in k.name) for s in long_)
        starts = sorted(min(k.time_range.start for k in by_stream[s] if "k_shard_select" in k.name) for s in short)
        assert all(a >= b for a, b in zip(starts, ends)), (starts, ends)
    finally:
        for e, a, b in zip(engs, h1, h2):
            e.release(a)
            e.release(b)
        _close(engs)


def test_two_handles_in_flight():
    _in_child("_in_flight", False)


def test_two_handles_in_flight_under_the_profiler():
    """Also in a process of its own for a second reason: a torch.profiler session sets up CUPTI for the whole process,
    and the tests that profile later in the same process (tests/test_gpu_chain.py's witnesses) must find it as if no
    other session had run before them."""
    _in_child("_in_flight", True)
