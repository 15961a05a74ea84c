"""GPU, ONE device: the node-axis sharding protocol with world = 2 and 4 contexts created on the
same GPU.  Replicated selection needs no collective at all; for the all-gather scheme the
per-rank key buffers (library-owned device memory) are concatenated with a device copy, which is
what the NCCL all-gather does between GPUs (tests/test_gpu_shard.py runs that on >= 2 GPUs).
Every rank's column slab of the dense matrix, the merged top-K lists and the placements are
compared bit for bit with the CPU oracle."""
import numpy as np
import pytest

from rbg_b200 import synth
from rbg_b200.engine import TopoPlacer

pytestmark = pytest.mark.gpu


class DevPtr:
    def __init__(self, p, nb):
        self.__cuda_array_interface__ = {"shape": (nb // 8,), "typestr": "<i8", "data": (p, False), "version": 3,
                                         "strides": None}


def _gather(ptrs):
    """All-gather of one device buffer per rank on a single GPU: concatenate, rank-major."""
    import torch
    torch.cuda.synchronize()
    parts = [torch.as_tensor(DevPtr(p, nb), device="cuda") for p, nb in ptrs]
    out = torch.cat(parts)
    torch.cuda.synchronize()
    return out


def _engines(topo, world):
    engs = []
    for r in range(world):
        e = TopoPlacer(device=0, rank=r, world=world)
        e.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
        engs.append(e)
    slabs = [e.slab() for e in engs]
    assert slabs[0][0] == 0 and slabs[-1][1] == topo.n and all(a[1] == b[0] for a, b in zip(slabs, slabs[1:]))
    return engs


@pytest.mark.parametrize("world", [2, 4])
def test_step_batches_sharded_on_one_device(world):
    from oracle import placer as oracle_placer
    from test_gpu_parity import _random_steps
    for n, seed, excl in [(4096, 1, False), (10000, 2, True), (3000, 3, True)]:
        topo = synth.make_topology(n, seed=seed, tiers=4, owned_frac=0.25 if excl else 0.0)
        blob = _random_steps(topo, 50 + seed, 24, excl=excl, gang=True)
        ref = oracle_placer.place(topo, blob)
        engs = _engines(topo, world)
        # ---- all-gather scheme
        hs = [e.stage(blob) for e in engs]
        allk = _gather([e.shard_score(h) for e, h in zip(engs, hs)])
        m = [e.shard_merge(h, allk.data_ptr()) for e, h in zip(engs, hs)]
        all2 = None
        if m[0][0]:
            assert all(x[0] for x in m)
            all2 = _gather([(x[1], x[2]) for x in m])
        for e, h in zip(engs, hs):
            e.shard_assign(h, all2.data_ptr() if all2 is not None else None)
        for r, (e, h) in enumerate(zip(engs, hs)):
            assign, status, domain = e.fetch(h)
            assert np.array_equal(assign, ref["assign"]), (world, r, n)
            assert np.array_equal(status, ref["status"]) and np.array_equal(domain, ref["domain"]), (world, r, n)
            lo, hi = e.slab()
            for row in range(0, ref["matrix"].shape[0], 5):
                got = e.read_scores(h, row)
                assert np.array_equal(got.view(np.uint32), ref["matrix"][row, lo:hi].view(np.uint32)), (world, r, row)
            for rr in range(ref["topk"].shape[0]):
                assert np.array_equal(e.read_topk(h, rr, 32), ref["topk"][rr]), (world, r, rr)
            e.release(h)
        # ---- replicated selection: no collective, plain run_staged / score_assign on every rank
        for r, e in enumerate(engs):
            h = e.stage(blob)
            e.run_staged(h, 1)
            a2, s2, d2 = e.fetch(h)
            assert np.array_equal(a2, ref["assign"]) and np.array_equal(s2, ref["status"]), (world, r, n)
            assert np.array_equal(d2, ref["domain"])
            lo, hi = e.slab()
            for row in range(0, ref["matrix"].shape[0], 7):
                got = e.read_scores(h, row)
                assert np.array_equal(got.view(np.uint32), ref["matrix"][row, lo:hi].view(np.uint32)), (world, r, row)
            for rr in range(ref["topk"].shape[0]):
                assert np.array_equal(e.read_topk(h, rr, 32), ref["topk"][rr]), (world, r, rr, "replicated")
            e.release(h)
            a3, s3, _ = e.score_assign(blob)
            assert np.array_equal(a3, ref["assign"]) and np.array_equal(s3, ref["status"])
        for e in engs:
            e.close()


@pytest.mark.parametrize("world", [2, 4])
def test_group_plans_sharded_on_one_device(world):
    from oracle import placer as oracle_placer
    from rbg_b200.blob import BlobBuilder
    from rbg_b200.plugin import B200TopoPodGroupManager, _GroupRun
    from test_gpu_groups import _fleet
    from test_plugin_host import OraclePlacer
    for n, kw in [(8000, {}), (6000, dict(excl_every=3, gang_every=4)), (5000, dict(big_every=5))]:
        topo = synth.make_topology(n, seed=n, tiers=4, owned_frac=0.2 if kw.get("excl_every") else 0.0)
        rbgs = _fleet(n, 24, seed=9, **kw)
        ref = B200TopoPodGroupManager(OraclePlacer(topo)).reconcile_pod_groups_by_waves(rbgs)
        engs = _engines(topo, world)
        gblob, runs = B200TopoPodGroupManager(engs[0]).groups_blob(rbgs)
        # ---- all-gather scheme, wave by wave
        hs = [e.stage_groups(gblob) for e in engs]
        for w in range(engs[0].shard_waves(hs[0])):
            allk = _gather([e.shard_wave_score(h, w) for e, h in zip(engs, hs)])
            m = [e.shard_wave_merge(h, w, allk.data_ptr()) for e, h in zip(engs, hs)]
            all2 = _gather([(x[1], x[2]) for x in m]) if m[0][0] else None
            for e, h in zip(engs, hs):
                e.shard_wave_assign(h, w, all2.data_ptr() if all2 is not None else None)
        res = [e.fetch(h) for e, h in zip(engs, hs)]
        for r, (assign, status, domain) in enumerate(res):
            off = 0
            for i, rr in enumerate(ref):
                want = list(rr.nodes.values())
                got = assign[off:off + len(want)].tolist()
                off += len(want)
                if rr.status == 1:   # the plan leaves non-gang partial groups to the host loop: status only
                    assert status[i] == 1, (world, r, n, i)
                    continue
                assert got == want, (world, r, n, i, got, want)
                assert status[i] == rr.status and domain[i] == rr.domain, (world, r, n, i)
        for e, h in zip(engs, hs):
            e.release(h)
        # ---- replicated selection on every rank + the host-buffer entry point
        for r, e in enumerate(engs):
            h = e.stage_groups(gblob)
            e.run_staged(h, 1)
            a2, s2, d2 = e.fetch(h)
            assert np.array_equal(a2, res[0][0]) and np.array_equal(s2, res[0][1]) and np.array_equal(d2, res[0][2]), (world, r, n)
            a4, s4, d4 = e.place_groups(gblob)
            off = 0
            for i, rr in enumerate(ref):
                want = list(rr.nodes.values())
                assert a4[off:off + len(want)].tolist() == want and s4[i] == rr.status and d4[i] == rr.domain, (world, r, n, i)
                off += len(want)
            if not kw:   # nobody fails in this fleet: the plan's rows line up with the wave-by-wave oracle run
                from gpu_util import plan_rows
                gruns = [_GroupRun(x, B200TopoPodGroupManager(e).arith) for x in rbgs]
                row_of = plan_rows(gblob, topo)
                index_of = {id(g): i for i, g in enumerate(gruns)}
                lo, hi = e.slab()
                w = 0
                while True:
                    active = [g for g in gruns if w < len(g.waves)]
                    if not active:
                        break
                    bb = BlobBuilder()
                    for g in active:
                        bb.add(g.step(w))
                    oref = oracle_placer.place(topo, bb.build(), want_matrix=True, want_topk=False)
                    assert oref["rc"] == 0 and (oref["status"] == 0).all()
                    off = 0
                    for i, g in enumerate(active):
                        cnt = sum(c for _, _, c in g.waves[w].roles)
                        row0 = row_of[(index_of[id(g)], w)]
                        for k in range(0, cnt, 2):
                            got = e.read_scores(h, row0 + k)
                            assert np.array_equal(got.view(np.uint32), oref["matrix"][off + k, lo:hi].view(np.uint32)), (world, r, w, i, k)
                        g.absorb(w, oref["assign"][off:off + cnt], int(oref["status"][i]), int(oref["domain"][i]), n)
                        off += cnt
                    w += 1
            e.release(h)
        for e in engs:
            e.close()
    # a generated fleet at the limits of the GROUPS ABI (8-role waves, 16-role groups, weighted pairs, N % 4 != 0)
    import groups_gen as gg
    from test_gpu_groups_limits import group_slices, oracle_plan
    case = gg.make_case(14, 2049)
    states, _ = oracle_plan(case.topo, case.blob)
    engs = _engines(case.topo, world)
    hs = [e.stage_groups(case.blob) for e in engs]
    for w in range(engs[0].shard_waves(hs[0])):
        allk = _gather([e.shard_wave_score(h, w) for e, h in zip(engs, hs)])
        m = [e.shard_wave_merge(h, w, allk.data_ptr()) for e, h in zip(engs, hs)]
        all2 = _gather([(x[1], x[2]) for x in m]) if m[0][0] else None
        for e, h in zip(engs, hs):
            e.shard_wave_assign(h, w, all2.data_ptr() if all2 is not None else None)
    res = [e.fetch(h) for e, h in zip(engs, hs)]
    for r, (assign, status, domain) in enumerate(res):
        for i, (st, sl) in enumerate(zip(states, group_slices(states))):
            want = st.result()
            if want["status"] == 1:   # left to the host loop by the plan: status only
                assert status[i] == 1, (world, r, i)
                continue
            assert assign[sl].tolist() == st.assign_in_group_order(), (world, r, i)
            assert (status[i], domain[i]) == (want["status"], want["domain"]), (world, r, i)
    for e, h in zip(engs, hs):
        e.release(h)
    for r, e in enumerate(engs):
        h = e.stage_groups(case.blob)
        e.run_staged(h, 1)
        a2, s2, d2 = e.fetch(h)
        assert np.array_equal(a2, res[0][0]) and np.array_equal(s2, res[0][1]) and np.array_equal(d2, res[0][2]), (world, r)
        e.release(h)
        a4, s4, d4 = e.place_groups(case.blob)
        for i, (st, sl) in enumerate(zip(states, group_slices(states))):
            want = st.result()
            assert a4[sl].tolist() == st.assign_in_group_order() and (s4[i], d4[i]) == (want["status"], want["domain"]), (world, r, i)
    for e in engs:
        e.close()


def _connect_p2p(engs):
    """Contexts of one process: exchange the raw device pointers of the exchange buffers."""
    ptrs = [e.p2p_export(rows_cap=4096)[1] for e in engs]
    for e in engs:
        e.p2p_import(ptrs=ptrs)


@pytest.mark.parametrize("world", [2, 4])
def test_p2p_allgather_inside_the_library(world):
    """rbgtopo_run_staged_p2p: the per-wave exchange of the rank-local lists done by the library's own
    kernels (peer stores + release/acquire flags), no collective library.  Same results as the oracle
    (step batches) / as replicated selection (plans), NVLink byte count reported, no timeout."""
    import torch
    from oracle import placer as oracle_placer
    from rbg_b200.plugin import B200TopoPodGroupManager
    from test_gpu_groups import _fleet
    from test_gpu_parity import _random_steps
    from test_plugin_host import OraclePlacer
    for n, seed, excl in [(4096, 1, False), (6000, 2, True)]:
        topo = synth.make_topology(n, seed=seed, tiers=4, owned_frac=0.25 if excl else 0.0)
        blob = _random_steps(topo, 70 + seed, 24, excl=excl, gang=True)
        ref = oracle_placer.place(topo, blob)
        engs = _engines(topo, world)
        _connect_p2p(engs)
        hs = [e.stage(blob) for e in engs]
        for rep in range(3):      # the parity / sequence bookkeeping survives repeated passes
            for e, h in zip(engs, hs):
                e.run_staged_p2p(h, 1)
        torch.cuda.synchronize()
        for r, (e, h) in enumerate(zip(engs, hs)):
            assign, status, domain = e.fetch(h)
            st = e.p2p_stats()
            assert not st["timed_out"] and st["peer_bytes_last_pass"] > 0, (world, r, st)
            assert np.array_equal(assign, ref["assign"]), (world, r, n)
            assert np.array_equal(status, ref["status"]) and np.array_equal(domain, ref["domain"]), (world, r, n)
            lo, hi = e.slab()
            for row in range(0, ref["matrix"].shape[0], 5):
                got = e.read_scores(h, row)
                assert np.array_equal(got.view(np.uint32), ref["matrix"][row, lo:hi].view(np.uint32)), (world, r, row)
            for rr in range(ref["topk"].shape[0]):
                assert np.array_equal(e.read_topk(h, rr, 32), ref["topk"][rr]), (world, r, rr)
            e.release(h)
        # whole groups: multi-wave plan through the p2p pipeline == replicated selection == oracle wave loop
        rbgs = _fleet(n, 24, seed=9, excl_every=3 if excl else 0, gang_every=4)
        oref = B200TopoPodGroupManager(OraclePlacer(topo)).reconcile_pod_groups_by_waves(rbgs)
        gblob, _ = B200TopoPodGroupManager(engs[0]).groups_blob(rbgs)
        hs = [e.stage_groups(gblob) for e in engs]
        for e, h in zip(engs, hs):
            e.run_staged_p2p(h, 1)
        torch.cuda.synchronize()
        res = [e.fetch(h) for e, h in zip(engs, hs)]
        for r, (e, h) in enumerate(zip(engs, hs)):
            assert not e.p2p_stats()["timed_out"]
            e.release(h)
            h2 = e.stage_groups(gblob)
            e.run_staged(h2, 1)
            rep_res = e.fetch(h2)
            e.release(h2)
            for x, y in zip(res[r], rep_res):
                assert np.array_equal(x, y), (world, r, n)
        off = 0
        for i, rr in enumerate(oref):
            want = list(rr.nodes.values())
            if rr.status != 1:   # non-gang partial groups are finished by the host loop, not by a staged plan
                assert res[0][0][off:off + len(want)].tolist() == want and res[0][1][i] == rr.status, (world, n, i)
            off += len(want)
        for e in engs:
            e.close()
