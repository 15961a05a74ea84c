"""CPU: every designed case of tests/test_gpu_shard_limits.py still hits its edge, before any GPU runs it
(tests/shard_limits_cases.py).  For every case at every world it names: its precondition holds on the world = 1
oracle; the numpy protocol models give the oracle's outputs — shard_rank (per-slab top lists, the rank-major merge)
for the one-pod ranked cases, the pod-job exchange for the leader-worker ones; and model_rows (the replicated
evaluator of k_lw_assign_repl) equals every dense row the oracle scores."""
import numpy as np
import pytest

import alternates_limits_cases as al
import lw_alternates_oracle as lwa
import shard_limits_cases as sc
from test_oracle_lw_shards import evaluator_checked, exchange  # noqa: F401  (a fixture)
from test_oracle_shard_alternates import slab_bounds


@pytest.mark.parametrize("name", sc.ALT_NAMES)
def test_alternates_case(evaluator_checked, name):
    _, worlds, n_alts, make = sc.alt_case(name)
    topo, gblob, pre = make()
    exp = pre()
    for W in worlds:
        for F in n_alts:
            got = sc.model_alternates(topo, gblob, exp, W, F)
            for r, alts in enumerate(got):
                assert alts == [int(m) for m in exp[4][r][:F] if m >= 0], (W, F, r, alts, exp[4][r])


@pytest.mark.parametrize("name", sc.LW_CASES)
def test_leader_worker_case(evaluator_checked, monkeypatch, name):
    topo, gblob, rp, pre = sc.lw_case(name)
    exp = pre()
    for W in sc.LW_WORLDS:
        monkeypatch.setattr(lwa, "ranked_candidates", exchange(slab_bounds(topo.n, W)))
        got = sc.lw_ranked_oracle(topo, gblob, rp)
        monkeypatch.undo()
        for x, y in zip(got, exp):
            x, y = np.asarray(x), np.asarray(y)
            assert np.array_equal(x.view(np.uint32) if x.dtype == np.float32 else x,
                                  y.view(np.uint32) if y.dtype == np.float32 else y), (name, W)


def test_committed_consumed_record_without_anchor(evaluator_checked):
    topo, gblob, rp, info = sc.committed_consumed_case()
    sc.committed_consumed_pre(topo, gblob, rp, info)
    sc.lw_ranked_oracle(topo, gblob, rp)         # the rows of the plain call through the evaluator


def test_helpers():
    assert sc.slab_thread_of(2176 + 1024 + 5, 2176) == 1 and sc.slab_thread_of(3000, 2176) == 206
    assert [sc.merge_lane_of(r, p) for r, p in [(0, 0), (3, 5), (7, 1), (10, 6), (14, 2)]] == [0] * 5
    assert sc.lane_keys(8, 0) == [(0, 0), (3, 5), (7, 1)]
    assert sc.lane_keys(16, 0) == [(0, 0), (3, 5), (7, 1), (10, 6), (14, 2)]
    assert slab_bounds(3000, 3) == [0, 896, 1920, 3000]
    assert slab_bounds(700, 8) == [0, 0, 128, 256, 256, 384, 512, 512, 700]
    assert al.merge_case("warp", "rank0")[1].tolist() == al.merge_case("warp", "rank0", 0, None)[1].tolist()
