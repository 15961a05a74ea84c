"""GPU: step-level batches (rbgtopo_score_assign, rbgtopo_stage + run_staged / read_scores / read_topk, and on world > 1
shard_score / shard_merge / shard_assign and run_staged_p2p) at the limits of the BLOB ABI, against the CPU oracle.

The batches come from tests/steps_gen.py: 8-role steps of 32 replicas (warps 5-7 of the 256-thread selection CTA, rows
5-7 of k_score_emit's role table), Q = 16, pair weights to 5, consumed amounts 0 and 32 767, duplicated consumed
nodes (summed in k_score_emit, in k_select_assign_fast's table and in the greedy), steps on both sides of
k_score_emit's two-record branch in one launch, every exclusive corner, ragged node counts from 1 to 4 097.  Batches
with one hub-anchored step take the global candidate list (k_select_assign at world 1, k_select on the all-gather
path); world 2 and 4 run on one device with empty slabs."""
import os
import subprocess
import sys

import numpy as np
import pytest

import steps_gen as sg
import topo_gen as tg
from gpu_util import check_batch, new_engine
from oracle import placer as oracle_placer
from rbg_b200 import synth
from rbg_b200.engine import RbgTopoError
from test_gpu_shard_single import _connect_p2p, _engines, _gather
from test_gpu_snapshot import _hubs_and_isolated

pytestmark = pytest.mark.gpu

ELIMIT, EINEXACT = -6, -4
FAST_SMEM_MAX = 200 * 1024      # shared memory of k_select_assign_fast / k_shard_select (kFastSmemMax)
CAND_CAP = 512                  # k_select_assign's shared candidate list and key cache (select.cuh)


def select_table(topo, steps):
    """(per-step patch capacities, CAP, HT) of the patched-node table of a step batch: CAP = max(32, round_up(largest
    capacity, 32)), HT = the smallest power of two >= 64 with 2·HT >= 3·CAP."""
    caps = [sg.patch_capacity(topo, s) for s in steps]
    cap = max(32, -(-max(caps) // 32) * 32)
    ht = 64
    while 2 * ht < 3 * cap:
        ht <<= 1
    return caps, cap, ht


def table_bytes(ht, cap, rows):
    """fast_smem_bytes: node and consumed slots, `rows` delta rows of HT floats, the dense view of CAP slots."""
    return ht * 4 * (2 + rows) + cap * 16


def fast_smem(topo, steps):
    """launch_select_assign's rule for a step batch: (per-step patch capacities, shared memory of the table).  The table
    has one delta row per warp of the CTA as launched, max(128, 32·P_max) threads; the batch takes k_select_assign_fast
    iff this fits FAST_SMEM_MAX, else the global candidate list."""
    caps, cap, ht = select_table(topo, steps)
    p_max = max(len(s.roles) for s in steps)
    return caps, table_bytes(ht, cap, max(4, p_max))


def _code(fn, *args):
    with pytest.raises(RbgTopoError) as ei:
        fn(*args)
    return ei.value.code


# ---------------------------------------------------------------- world 1
@pytest.mark.parametrize("seed,n,ns", sg.CASES)
def test_world1_generated_batches(seed, n, ns):
    case = sg.make_case(seed, n, ns)
    eng = new_engine(case.topo)
    try:
        check_batch(eng, case.topo, case.blob)
    finally:
        eng.close()


def test_world1_chunked_node_axis():
    """chunk_nodes = 128 at N = 4 097: 33 chunks per row, the last one a single ragged node."""
    case = sg.make_case(8, 4097, 33)
    eng = new_engine(case.topo, chunk_nodes=128)
    try:
        check_batch(eng, case.topo, case.blob)
    finally:
        eng.close()


@pytest.mark.parametrize("name", ["hubs", "big_hub"])
def test_world1_global_candidate_list(name):
    """One hub-anchored step among small ones: its patch capacity puts the whole batch past k_select_assign_fast's
    shared memory, so every step runs k_select_assign — the small ones with the shared candidate list and cached
    keys, the heavy one with the global scratch and uncached keys — reading the patched scores back from the matrix
    k_score_emit corrected."""
    topo = tg.make(name).topo
    steps = sg.hub_batch(topo, 5)
    caps, smem = fast_smem(topo, steps)
    heavy = len(steps) // 2
    assert smem > FAST_SMEM_MAX, smem
    assert caps[heavy] > 10 * CAND_CAP and all(c <= CAND_CAP for i, c in enumerate(caps) if i != heavy), caps
    assert max(len(s.roles) for s in steps) >= 6
    eng = new_engine(topo)
    try:
        check_batch(eng, topo, sg.build(steps))
    finally:
        eng.close()


def _few_role_batch(topo, max_roles):
    """A batch of 1..max_roles-role steps, one of them with enough records on the hub that a table with one delta row
    per ROLE would fit FAST_SMEM_MAX while the table of the 4-warp CTA actually launched does not."""
    for k in range(1, 400):
        steps = sg.hub_batch(topo, 7, hub_records=k, max_roles=max_roles)
        _, cap, ht = select_table(topo, steps)
        p_max = max(len(s.roles) for s in steps)
        if table_bytes(ht, cap, p_max) <= FAST_SMEM_MAX < table_bytes(ht, cap, max(4, p_max)):
            assert p_max <= max_roles and fast_smem(topo, steps)[1] > FAST_SMEM_MAX
            return steps
    raise AssertionError("no few-role batch between the two table sizes")


@pytest.mark.parametrize("max_roles", [1, 2])
def test_world1_few_role_batch_past_the_launched_table(max_roles):
    """Steps of at most 2 roles on a synth cluster (degree <= 42), one of them with a patch capacity of a few thousand:
    the batch takes the global candidate list and places what the oracle places.  Sizing the fast kernel's table by
    the roles instead of the launched warps sent such a batch to a k_select_assign_fast launch past its shared memory
    (RBGTOPO_ECUDA for a valid batch)."""
    topo = synth.make_topology(4096, seed=3, tiers=4)
    steps = _few_role_batch(topo, max_roles)
    eng = new_engine(topo)
    try:
        check_batch(eng, topo, sg.build(steps))
    finally:
        eng.close()


def test_sharded_few_role_batch_past_the_launched_table():
    """The same batch on two ranks: the all-gather calls take k_select with parity, replicated selection refuses it with
    RBGTOPO_ELIMIT (the documented limit, not a failed launch) and the contexts stay usable."""
    topo = synth.make_topology(4096, seed=3, tiers=4)
    blob = sg.build(_few_role_batch(topo, 2))
    ref = oracle_placer.place(topo, blob)
    assert ref["rc"] == 0
    small = sg.build(sg.hub_batch(topo, 7, max_roles=2))
    sref = oracle_placer.place(topo, small)
    engs = _engines(topo, 2)
    try:
        _all_gather(engs, blob, ref, ("few roles",))
        for r, e in enumerate(engs):
            h = e.stage(blob)
            try:
                assert _code(e.run_staged, h, 1) == ELIMIT, r
            finally:
                e.release(h)
            assert _code(e.score_assign, blob) == ELIMIT, r
        _replicated(engs, small, sref, ("few roles, small",))
    finally:
        for e in engs:
            e.close()


def test_world1_exactness_edge():
    """A role at need·8 + Σ pair·count = 1 118 on a snapshot whose rows all sum to 7 000: admitted, scores in
    [2^23, 2^24) with bit parity; one more pod is -4 from score_assign and stage, and the context stays usable."""
    topo, steps = sg.exactness_edge()
    _, over = sg.exactness_edge(1)
    ok, bad = sg.build(steps), sg.build(over)
    eng = new_engine(topo)
    try:
        ref = check_batch(eng, topo, ok)
        assert 2 ** 23 <= float(ref["matrix"].max()) < 2 ** 24
        for f in (eng.score_assign, eng.stage):
            assert _code(f, bad) == EINEXACT
        check_batch(eng, topo, ok, ref=ref)
    finally:
        eng.close()


# ---------------------------------------------------------------- world 2 / 4 on one device
def _check_rank(e, h, ref, tag):
    """This rank's slab of every dense row, the merged top-K of every role row, the placements."""
    assign, status, domain = e.fetch(h)
    assert np.array_equal(assign, ref["assign"]), tag
    assert np.array_equal(status, ref["status"]) and np.array_equal(domain, ref["domain"]), tag
    lo, hi = e.slab()
    for row in range(ref["matrix"].shape[0]):
        got = e.read_scores(h, row)
        assert len(got) == hi - lo
        assert np.array_equal(got.view(np.uint32), ref["matrix"][row, lo:hi].view(np.uint32)), tag + ("row", row)
    for rr in range(ref["topk"].shape[0]):
        assert np.array_equal(e.read_topk(h, rr, 32), ref["topk"][rr]), tag + ("topk", rr)


def _all_gather(engs, blob, ref, tag):
    hs = [e.stage(blob) for e in engs]
    try:
        allk = _gather([e.shard_score(h) for e, h in zip(engs, hs)])
        m = [e.shard_merge(h, allk.data_ptr()) for e, h in zip(engs, hs)]
        all2 = None
        if m[0][0]:
            assert all(x[0] for x in m)
            all2 = _gather([(x[1], x[2]) for x in m])
        for e, h in zip(engs, hs):
            e.shard_assign(h, all2.data_ptr() if all2 is not None else None)
        for r, (e, h) in enumerate(zip(engs, hs)):
            _check_rank(e, h, ref, tag + ("all-gather", r))
    finally:
        for e, h in zip(engs, hs):
            e.release(h)


def _replicated(engs, blob, ref, tag):
    for r, e in enumerate(engs):
        h = e.stage(blob)
        try:
            e.run_staged(h, 1)
            _check_rank(e, h, ref, tag + ("replicated", r))
        finally:
            e.release(h)
        a, s, d = e.score_assign(blob)
        assert np.array_equal(a, ref["assign"]) and np.array_equal(s, ref["status"]) and np.array_equal(d, ref["domain"]), tag + (r,)


def _p2p(engs, blob, ref, tag):
    import torch
    hs = [e.stage(blob) for e in engs]
    try:
        for e, h in zip(engs, hs):
            e.run_staged_p2p(h, 1)
        torch.cuda.synchronize()
        for r, (e, h) in enumerate(zip(engs, hs)):
            assert not e.p2p_stats()["timed_out"], tag + (r,)
            _check_rank(e, h, ref, tag + ("p2p", r))
    finally:
        for e, h in zip(engs, hs):
            e.release(h)


def _heavy_batch(topo, seed):
    """hub_batch with as many records on the hub as it takes to put the batch past the table's shared memory."""
    for k in range(1, 1000):
        steps = sg.hub_batch(topo, seed, hub_records=k)
        caps, smem = fast_smem(topo, steps)
        if smem > FAST_SMEM_MAX:
            return steps
    raise AssertionError("no hub batch past the shared-memory limit")


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("seed,n", [(21, 100), (22, 300)])
def test_sharded_step_batches_on_one_device(world, seed, n):
    case = sg.make_case(seed, n, 17)
    topo = case.topo
    ref = oracle_placer.place(topo, case.blob)
    assert ref["rc"] == 0
    heavy = sg.build(_heavy_batch(topo, seed))
    href = oracle_placer.place(topo, heavy)
    assert href["rc"] == 0
    engs = _engines(topo, world)
    try:
        slabs = [e.slab() for e in engs]
        # slab bounds are multiples of 128: at N = 100 and at N = 300 over 4 ranks some rank has nothing to score
        assert any(lo == hi for lo, hi in slabs) == (n == 100 or world == 4), slabs
        if n == 300:                                                       # the hub's neighbours on both sides of a slab boundary
            hub = _hubs_and_isolated(topo, 1)[0][0]
            nb = topo.col_idx[topo.row_ptr[hub]:topo.row_ptr[hub + 1]]
            assert any((nb < lo).any() and (nb >= lo).any() for lo, _ in slabs if 0 < lo < n), slabs
        _connect_p2p(engs)
        tag = (world, n)
        _all_gather(engs, case.blob, ref, tag)
        _replicated(engs, case.blob, ref, tag)
        _p2p(engs, case.blob, ref, tag)
        # the hub-anchored batch: the all-gather calls take k_select (global candidate list) ...
        _all_gather(engs, heavy, href, tag + ("heavy",))
        # ... replicated selection and the in-library exchange refuse it, and the contexts stay usable
        for r, e in enumerate(engs):
            h = e.stage(heavy)
            try:
                assert _code(e.run_staged, h, 1) == ELIMIT, (tag, r)
            finally:
                e.release(h)
            assert _code(e.score_assign, heavy) == ELIMIT, (tag, r)
            a, s, d = e.score_assign(case.blob)
            assert np.array_equal(a, ref["assign"]) and np.array_equal(s, ref["status"]), (tag, r)
            assert np.array_equal(d, ref["domain"]), (tag, r)
        hs = [e.stage(heavy) for e in engs]
        try:
            for r, (e, h) in enumerate(zip(engs, hs)):
                assert _code(e.run_staged_p2p, h, 1) == ELIMIT, (tag, r)
        finally:
            for e, h in zip(engs, hs):
                e.release(h)
        _p2p(engs, case.blob, ref, tag + ("after ELIMIT",))
    finally:
        for e in engs:
            e.close()


# ---------------------------------------------------------------- k_score_emit's step block at both limits
@pytest.mark.parametrize("block", ["1", "16"])
def test_emit_block_variants_in_a_subprocess(block):
    """The library reads RBGTOPO_EMIT_BLOCK when it loads, hence the subprocess: the world-1 tests above with
    k_score_emit staging 1 and 16 steps per CTA (EMIT_MAX_BLOCK) instead of 4."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, RBGTOPO_EMIT_BLOCK=block)
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "gpu", "-x",
                        "tests/test_gpu_steps_limits.py", "-k", "world1"],
                       cwd=root, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert "passed" in r.stdout
