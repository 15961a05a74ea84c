"""CPU: the seeded step-batch generator of the limit tests (tests/steps_gen.py) reaches what it claims to reach, and the
CPU references agree on it.  Its seed set must cover every limit in steps_gen.BULLETS (status and D* as the oracle
computes them), every step must stay under validate_blob's exactness bound, and the C oracle, its parallel variant
with the GPU path's algebra and the numpy restatement must agree bit for bit — so tests/test_gpu_steps_limits.py can
use the oracle as its reference at these limits."""
import numpy as np
import pytest

import steps_gen as sg
from oracle import placer, placer_ref
from rbg_b200.blob import STEP_EXCLUSIVE


def _same(a, b, tag):
    assert a["rc"] == 0 and b.get("rc", 0) == 0, (tag, a["rc"], b.get("rc"))
    assert np.array_equal(a["matrix"].view(np.uint32), b["matrix"].view(np.uint32)), tag
    assert np.array_equal(a["topk"], b["topk"]), tag
    assert np.array_equal(a["assign"], b["assign"]), tag
    assert np.array_equal(a["status"], b["status"]), tag
    assert np.array_equal(a["domain"], b["domain"]), tag


def test_generated_cases_cover_the_abi_limits():
    covered = dict.fromkeys(sg.BULLETS, False)
    for seed, n, ns in sg.CASES:
        case = sg.make_case(seed, n, ns)
        limit = sg.amax_limit(case.topo)
        assert all(sg.exact_ok(s, limit) for s in case.steps), seed
        ref = placer.place(case.topo, case.blob, want_matrix=False, want_topk=False)
        assert ref["rc"] == 0, (seed, ref["rc"])
        for si, s in enumerate(case.steps):
            if not s.flags & STEP_EXCLUSIVE:
                assert ref["domain"][si] == -1, (seed, si)      # a fixed domain on a non-exclusive step is not reported
        for k, v in sg.coverage(case, ref).items():
            covered[k] |= v
    assert all(covered.values()), [k for k, v in covered.items() if not v]


@pytest.mark.parametrize("seed,n,ns", sg.CASES)
def test_cpu_references_agree(seed, n, ns):
    case = sg.make_case(seed, n, ns)
    a = placer.place(case.topo, case.blob)
    for threads in (1, 4):
        _same(a, placer.place_fast(case.topo, case.blob, nthreads=threads), ("fast", threads))
    if n <= 300:
        _same(a, placer_ref.place(case.topo, case.blob), "ref")


def test_hub_batch_references_agree():
    topo, _, _ = sg.topology(22, 300)
    steps = sg.hub_batch(topo, 22, hub_records=40)
    blob = sg.build(steps)
    a = placer.place(topo, blob)
    _same(a, placer.place_fast(topo, blob, nthreads=4), "fast")
    _same(a, placer_ref.place(topo, blob), "ref")


def test_exactness_edge_sits_on_the_bound():
    topo, steps = sg.exactness_edge()
    limit = sg.amax_limit(topo)
    assert limit == 1119 and sg.role_mass(steps[0], 0) == limit - 1
    assert sg.exact_ok(steps[0], limit)
    blob = sg.build(steps)
    a = placer.place(topo, blob)
    assert a["rc"] == 0
    assert 2 ** 23 <= float(a["matrix"].max()) < 2 ** 24
    _same(a, placer.place_fast(topo, blob), "fast")
    _same(a, placer_ref.place(topo, blob), "ref")
    _, over = sg.exactness_edge(1)
    assert not sg.exact_ok(over[0], limit)


def test_generator_is_deterministic():
    a, b = sg.make_case(6, 130, 33), sg.make_case(6, 130, 33)
    assert (a.blob == b.blob).all() and (a.topo.domain_owner == b.topo.domain_owner).all()
    assert (a.topo.free == b.topo.free).all() and (a.topo.col_idx == b.topo.col_idx).all()
