"""GPU, one device: the rbgtopo_set_stream contract.

Every entry point on a caller stream (a torch.cuda.Stream, and the legacy default stream) with a bounded sleep queued
ahead of it, bit for bit against an internal-stream context and the oracle; snapshot refreshes issued while a pass is
still queued on the caller stream; and work that crosses a stream switch: whatever was enqueued before
rbgtopo_set_stream must be ordered before what is enqueued after it, whichever streams the two sides use."""
import os
import subprocess
import sys

import numpy as np
import pytest

import groups_gen as gg
import lw_commit_gen as lg
import lw_commit_levels_gen as lvg
import steps_gen as sg
from gpu_util import assert_same_result, check_batch, new_engine, plan_result, sleep_on
from rbg_b200 import synth
from test_gpu_groups_limits import check_direct, check_handle, check_staged, defined_rows, oracle_plan

pytestmark = pytest.mark.gpu


def _stream(kind):
    """(torch stream to queue on, handle for set_stream): a new stream, or torch's default (the legacy stream, 0)."""
    import torch
    if kind == "legacy":
        return torch.cuda.default_stream(), 0
    st = torch.cuda.Stream()
    return st, st.cuda_stream


def _bits(x):
    x = np.asarray(x)
    return x.view(np.uint32) if x.dtype == np.float32 else x


def _same(got, exp, tag):
    if not isinstance(got, tuple):
        got, exp = (got,), (exp,)
    for i, (x, y) in enumerate(zip(got, exp)):
        assert np.array_equal(_bits(x), _bits(y)), (tag, i, np.nonzero(_bits(x) != _bits(y))[0][:8])


def _both(calls, ie, ce, st, tag):
    """Each call on the caller-stream context behind a sleep (the call's own oracle check runs there), then on the
    internal-stream context; their outputs bit-identical."""
    for name, f in calls:
        sleep_on(st)
        got = f(ce)
        exp = f(ie)
        _same(got, exp, (tag, name))


def _entry_points_case(kind, tag):
    import test_gpu_alternates as ta
    import test_gpu_committed as tc
    import test_gpu_committed_alternates as tca
    import test_gpu_lw as tl
    import test_gpu_lw_alternates as tla
    import test_gpu_lw_committed as tlc
    import test_gpu_lw_committed_alternates as tlca
    import test_gpu_lw_committed_levels as tlcl
    st, handle = _stream(kind)

    def pair(topo, make=new_engine):
        ie, ce = make(topo), make(topo)
        ce.set_stream(handle)
        return ie, ce

    # step batches: stage / run_staged / fetch / read_scores / read_topk, then score_assign (check_batch)
    from oracle import placer as oracle_placer
    sc = sg.make_case(*sg.CASES[6])
    sref = oracle_placer.place(sc.topo, sc.blob, want_matrix=True, want_topk=True)   # before the sleep: the library's
    ie, ce = pair(sc.topo)                                                            # calls are what queue behind it
    try:
        def steps(e):
            check_batch(e, sc.topo, sc.blob, ref=sref)
            return e.score_assign(sc.blob)
        _both([("steps", steps)], ie, ce, st, tag)
        # GROUPS entry points on one fleet
        case = gg.make_case(5, 2049, n_groups=10)
        topo, gb = case.topo, case.blob
        states, waves = oracle_plan(topo, gb)
        rp = tl.cycle_pods(gb)
        ie.close()
        ce.close()
        ie, ce = pair(topo)

        def direct(e):
            check_direct(e, states, gb)
            return e.place_groups(gb)

        def staged(e):
            check_staged(e, topo, states, waves, gb)
            return e.place_groups(gb)
        calls = [("place_groups", direct), ("staged", staged),
                 ("committed", lambda e: tc.check(e, topo, gb, fast=True)),
                 ("committed_ranked", lambda e: tca.check(e, topo, gb, 3)),
                 ("ranked", lambda e: ta.check(e, topo, gb, 3)),
                 ("lw", lambda e: tl.check(e, topo, gb, rp)),
                 ("lw_ranked", lambda e: tla.check(e, topo, gb, rp, 3))]
        _both(calls, ie, ce, st, tag)
        ie.close()
        ce.close()
        # committed leader-worker batches, plain context
        f = lg.fleet(4, 130, scarce=True)
        ie, ce = pair(f.topo)
        fb, frp = f.blob(), f.role_pods()
        _both([("lw_committed", lambda e: tlc.check(e, f.topo, fb, frp)),
               ("lw_committed_ranked", lambda e: tlca.check(e, f.topo, fb, frp, n_alts=(3,)))], ie, ce, st, tag)
        ie.close()
        ce.close()
        # ... and on a lw_committed_levels context
        lf = lvg.fleet(4, 130, scarce=True, kind="mixed")
        ie, ce = tlcl.lv_engine(lf), tlcl.lv_engine(lf)
        ce.set_stream(handle)
        _both([("lw_committed_levels", lambda e: tlcl.check(e, lf)),
               ("lw_committed_levels_ranked", lambda e: e.place_groups_lw_committed_ranked(lf.blob(), lf.role_pods(), 3))],
              ie, ce, st, tag)
        # back to the internal streams: the next calls are unchanged
        ce.set_stream(None)
        _same(tlcl.check(ce, lf), tlcl.check(ie, lf), (tag, "after set_stream(None)"))
        _same(ce.place_groups_lw_committed_ranked(lf.blob(), lf.role_pods(), 3),
              ie.place_groups_lw_committed_ranked(lf.blob(), lf.role_pods(), 3), (tag, "ranked after set_stream(None)"))
    finally:
        ie.close()
        ce.close()


@pytest.mark.parametrize("kind", ["stream", "legacy"])
def test_every_entry_point_on_a_caller_stream(kind):
    _entry_points_case(kind, kind)


@pytest.mark.parametrize("var", ["RBGTOPO_SPLIT_MIN_GROUPS", "RBGTOPO_NO_DIRECT"])
def test_entry_points_on_other_paths_in_a_subprocess(var):
    """RBGTOPO_SPLIT_MIN_GROUPS=1 (-> 2): place_groups pipelines the fleet as two halves (ev[2] and stream2 beside the
    caller stream); RBGTOPO_NO_DIRECT: place_groups through the staged path (expanded plan, early emit on stream2)."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ)
    env[var] = "1"
    r = subprocess.run([sys.executable, "-m", "pytest", "tests/test_gpu_caller_stream.py", "-q", "-m", "gpu", "-x",
                        "-k", "test_every_entry_point"], cwd=root, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert "passed" in r.stdout


def _fleet(seed=6, n=4097):
    case = gg.make_case(seed, n, n_groups=12, scarce=True)
    return case.topo, case.blob


def _with_free(topo, free):
    return synth.Topology(topo.row_ptr, topo.col_idx, topo.edge_w, np.asarray(free, dtype=np.int32), topo.domain,
                          topo.domain_owner)


def test_refreshes_behind_queued_work():
    """run_staged (and a chain) queued behind a sleep on the caller stream, then update_nodes, then update_nodes_delta:
    fetch shows the OLD snapshot's results, bit for bit with the oracle, the next pass the new one's."""
    import torch
    topo, gb = _fleet()
    n = topo.n
    rng = np.random.default_rng(3)
    free2 = np.where(rng.random(n) < 0.3, 0, topo.free).astype(np.int32)
    nodes = np.sort(rng.choice(n, size=40, replace=False)).astype(np.int32)
    free3 = free2.copy()
    free3[nodes] = (free2[nodes] + 1) % 5
    snaps = [topo, _with_free(topo, free2), _with_free(topo, free3)]
    plans = [oracle_plan(t, gb) for t in snaps]
    eng = new_engine(topo)
    st = torch.cuda.Stream()
    eng.set_stream(st.cuda_stream)
    try:
        h, h2 = eng.stage_groups(gb), eng.stage_groups(gb)
        refresh = [lambda: eng.update_nodes(free2, None, generation=2),
                   lambda: eng.update_nodes_delta(nodes, free3[nodes], generation=3)]
        for k, upd in enumerate(refresh):
            sleep_on(st)
            eng.run_staged(h, 1)
            eng.run_staged_chain([h2, h], 5)
            upd()
            for x in (h, h2):
                check_handle(eng, topo, *plans[k], gb, x)
            eng.run_staged(h, 1)
            check_handle(eng, topo, *plans[k + 1], gb, h)
        eng.release(h)
        eng.release(h2)
    finally:
        eng.close()


def test_occupancy_refresh_behind_queued_work():
    """set_exclusive_levels with new records on the installed partitions fences without a host sync: the pass queued
    before it places with the old owners, the next one with the new (placements against the oracle on each group's
    level view)."""
    import torch
    import levels_oracle as lo
    import levels_view as lvw
    from test_gpu_levels_place import assert_fleet, engine, fleet
    topo, lv, nd, gb, occ = fleet(45, 2049, "random", scarce=True)
    occ2 = lo.random_occ(np.random.default_rng(9), topo.n, 3, [int(gb[8]), int(gb[8 + 12]), 998], max(1, topo.n // 5))
    exp1, _ = lvw.expected_fleet(topo, lv, lo.derive_level_owner(lv, occ), nd, gb)
    exp2, _ = lvw.expected_fleet(topo, lv, lo.derive_level_owner(lv, occ2), nd, gb)
    eng = engine(topo)
    st = torch.cuda.Stream()
    try:
        eng.set_exclusive_levels(lv[1:], occ, level_n_domains=nd[1:])
        eng.set_stream(st.cuda_stream)
        h = eng.stage_groups(gb)
        sleep_on(st)
        eng.run_staged(h, 1)
        eng.set_exclusive_levels(None, occ2)
        assert_fleet(eng.fetch(h), exp1, gb, "queued before the refresh", staged=True)
        eng.run_staged(h, 1)
        assert_fleet(eng.fetch(h), exp2, gb, "after the refresh", staged=True)
        eng.release(h)
    finally:
        eng.close()


CROSS = ["a_internal_fetch", "b_other_stream_fetch", "c_update_nodes", "d_rerun_on_other_stream", "e_internal_to_caller",
         "c_set_topology", "c_partition_install"]


@pytest.mark.parametrize("case", CROSS)
def test_work_that_crosses_a_switch(case):
    """A sleep and a run_staged on stream A, then (a) set_stream(None) and fetch / read_scores, (b) set_stream(B) and
    fetch, (c) set_stream(None), a refresh, fetch — the old snapshot's results (update_nodes; set_topology, after which
    the handle is stale and a new one sees the new topology; a partition install, which keeps level-0 handles), (d)
    set_stream(B) and run_staged of the same handle of bench.py's fleet, B having a sleep of its own queued as long as
    A's, so that without the switch's ordering the two passes of one matrix would run at once: exactly one pass's rows,
    and (e) the reverse: many passes on the internal streams, then set_stream(A) and fetch."""
    import torch
    topo, gb = _fleet()
    states, waves = oracle_plan(topo, gb)
    sel = defined_rows(topo, states, waves, gb)
    want = None
    if case == "d_rerun_on_other_stream":
        # bench.py's fleet: a pass long enough (~0.1 ms) that two unordered passes started together overlap.  The expected
        # rows come first, before anything is queued: closing a context synchronises the device.
        from test_gpu_chain import bench_fleet
        topo, _, gb, sel = bench_fleet()
        ref = new_engine(topo)
        r = ref.stage_groups(gb)
        ref.run_staged(r, 1)
        want = plan_result(ref, r, *sel)
        ref.close()
    eng = new_engine(topo)
    A, B = torch.cuda.Stream(), torch.cuda.Stream()
    try:
        if case == "e_internal_to_caller":
            h = eng.stage_groups(gb)
            eng.run_staged(h, 200)   # a fresh handle: nothing valid in its output buffers until a pass ends
            eng.set_stream(A.cuda_stream)
            check_handle(eng, topo, states, waves, gb, h)
            return
        eng.set_stream(A.cuda_stream)
        h = eng.stage_groups(gb)
        if case == "d_rerun_on_other_stream":
            sleep_on(B)   # B's own earlier work, as long as A's: unordered, the two passes would start together
        sleep_on(A)
        eng.run_staged(h, 1)
        if case == "a_internal_fetch":
            eng.set_stream(None)
            check_handle(eng, topo, states, waves, gb, h)
        elif case == "b_other_stream_fetch":
            eng.set_stream(B.cuda_stream)
            check_handle(eng, topo, states, waves, gb, h)
        elif case == "c_update_nodes":
            eng.set_stream(None)
            free2 = np.where(np.arange(topo.n) % 3 == 0, 0, topo.free).astype(np.int32)
            eng.update_nodes(free2, None, generation=5)
            check_handle(eng, topo, states, waves, gb, h)
            eng.run_staged(h, 1)
            check_handle(eng, topo, *oracle_plan(_with_free(topo, free2), gb), gb, h)
        elif case == "d_rerun_on_other_stream":
            eng.set_stream(B.cuda_stream)
            eng.run_staged(h, 1)
            assert_same_result(plan_result(eng, h, *sel), want, "two passes, one after the other")
        elif case == "c_set_topology":
            eng.set_stream(None)
            free2 = np.where(np.arange(topo.n) % 2 == 0, topo.free, 0).astype(np.int32)
            eng.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, free2, topo.domain, topo.domain_owner)
            with pytest.raises(Exception):
                eng.fetch(h)        # stale: the topology changed
            h2 = eng.stage_groups(gb)
            eng.run_staged(h2, 1)
            check_handle(eng, topo, *oracle_plan(_with_free(topo, free2), gb), gb, h2)
        elif case == "c_partition_install":
            eng.set_stream(None)
            lv = np.stack([np.arange(topo.n), np.zeros(topo.n, np.int64)]).astype(np.int32)
            eng.set_exclusive_levels(lv, np.zeros((0, 3), np.int32))
            check_handle(eng, topo, states, waves, gb, h)   # level-0 handle: kept, the pass before the install
            eng.run_staged(h, 1)
            ref = new_engine(topo)
            ref.set_exclusive_levels(lv, np.zeros((0, 3), np.int32))
            r = ref.stage_groups(gb)
            ref.run_staged(r, 1)
            want = plan_result(ref, r, *sel)
            ref.close()
            assert_same_result(plan_result(eng, h, *sel), want, "after the install")
    finally:
        torch.cuda.synchronize()   # nothing of the case is left running when its context goes
        eng.close()
