"""Shared helpers of the GPU parity tests (test infrastructure)."""
import numpy as np

from oracle import placer as oracle_placer
from rbg_b200.engine import TopoPlacer


def new_engine(topo, **kw):
    eng = TopoPlacer(device=0, **kw)
    eng.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    return eng


def check_batch(eng, topo, blob, check_matrix=True, check_topk=True, ref=None):
    """Run blob on the GPU through the C ABI and on the oracle; assert bit-equality
    of the dense matrix, the final top-K keys, the assignment, status and domain."""
    if ref is None:
        ref = oracle_placer.place(topo, blob, want_matrix=check_matrix, want_topk=check_topk)
    assert ref["rc"] == 0, ref["rc"]
    h = eng.stage(blob)
    try:
        eng.run_staged(h, 1)
        assign, status, domain = eng.fetch(h)
        if check_matrix:
            for row in range(ref["matrix"].shape[0]):
                got = eng.read_scores(h, row)
                exp = ref["matrix"][row]
                if not np.array_equal(got.view(np.uint32), exp.view(np.uint32)):
                    bad = np.nonzero(got.view(np.uint32) != exp.view(np.uint32))[0]
                    raise AssertionError(f"matrix row {row}: {len(bad)} mismatches, first at node {bad[0]}: "
                                         f"gpu={got[bad[0]]} oracle={exp[bad[0]]}")
        if check_topk:
            for rr in range(ref["topk"].shape[0]):
                got = eng.read_topk(h, rr, 32)
                assert np.array_equal(got, ref["topk"][rr]), (rr, got[:8], ref["topk"][rr][:8])
        assert np.array_equal(assign, ref["assign"]), (assign[:32], ref["assign"][:32])
        assert np.array_equal(status, ref["status"])
        assert np.array_equal(domain, ref["domain"])
    finally:
        eng.release(h)
    # and through the host-buffer entry point
    a2, s2, d2 = eng.score_assign(blob)
    assert np.array_equal(a2, ref["assign"]) and np.array_equal(s2, ref["status"]) and np.array_equal(d2, ref["domain"])
    return ref


# ~50 ms of GPU time at H100 clocks: long enough that a host enqueues a whole call sequence behind it, short enough
# to queue once per case
SLEEP_CYCLES = 100_000_000


def sleep_on(stream, cycles=SLEEP_CYCLES):
    """Queue a bounded busy kernel on `stream` (a torch.cuda.Stream; None: torch's default, the legacy stream)."""
    import torch
    with torch.cuda.stream(stream if stream is not None else torch.cuda.default_stream()):
        torch.cuda._sleep(int(cycles))


def plan_result(eng, h, rows, roles):
    """What a staged GROUPS handle exposes after its last pass: (assign, status, domain, the dense rows of the replica
    rows `rows` as float32 bits [len(rows)][slab], the 32 top-K keys of the role rows `roles` [len(roles)][32])."""
    a, s, d = eng.fetch(h)
    lo, hi = eng.slab()
    m = np.zeros((len(rows), hi - lo), dtype=np.uint32)
    for i, r in enumerate(rows):
        m[i] = eng.read_scores(h, r).view(np.uint32)
    topk = np.zeros((len(roles), 32), dtype=np.uint64)
    for i, p in enumerate(roles):
        topk[i] = eng.read_topk(h, p, 32)
    return a.copy(), s.copy(), d.copy(), m, topk


def assert_same_result(got, exp, tag):
    """Bit equality of two plan_result tuples, naming the first differing output and element."""
    for name, x, y in zip(("assign", "status", "domain", "rows", "topk"), got, exp):
        assert x.shape == y.shape, (tag, name, x.shape, y.shape)
        bad = np.argwhere(x != y)
        assert len(bad) == 0, (tag, name, f"{len(bad)} differ, first at {tuple(int(v) for v in bad[0])}",
                               x[tuple(bad[0])], y[tuple(bad[0])])


def plan_rows(gblob, topo):
    """(group, wave) -> dense-matrix row of the wave's first replica in a staged multi-wave plan
    (rows are in GROUP order: a group's waves are consecutive; rbgtopo_plan_describe column 4)."""
    from rbg_b200.engine import plan_steps
    return {(int(st[0]), int(st[1])): int(st[4]) for st in plan_steps(gblob, topo.n, len(topo.domain_owner))}
