"""GPU: dense matrices past 2^31 elements, with the boundary inside a row (tests/wide_matrix_cases.py).

Every kernel that touches the dense matrix forms a row's address as (size_t)row * slab_stride: k_emit_rows,
k_plan_group's corrections and k_plan_correct, k_score_emit, k_select_assign's read-back, k_alternates, k_lw_assign,
and on the host rbgtopo_read_scores and the kept rows of the ranked host-driven loops.  Were one of them an int
product, the upper part of a row would land elsewhere in the buffer, and since DevBuf::reserve allocates 1.25x what
is asked the stray store could stay in bounds.  Here 7 200 role rows at N = 300 000 (about 8.1 GiB of floats) go
through every entry point in both chunk configurations, and every output is compared bit for bit with the oracles:
every row read back with read_scores where a handle exists, the ranked outputs (score bits and alternates) where not.

Each case first checks torch.cuda.mem_get_info() and skips, naming what it needed and what was free.  At most one
wide context exists at a time and every context is closed in `finally`."""
import os
import subprocess
import sys

import numpy as np
import pytest

import wide_matrix_cases as wm
from rbg_b200.engine import plan_steps

pytestmark = pytest.mark.gpu

ROWS = wm.G * wm.Q
CHUNK_IDS = ["default", "chunk1920"]
# switches under which place_groups leaves the direct path, or runs it as two halves
SWITCHES_OFF_DIRECT = ("RBGTOPO_NO_DIRECT", "RBGTOPO_PER_WAVE_PLAN", "RBGTOPO_SPLIT_MIN_GROUPS", "RBGTOPO_CONCURRENT_PLAN")
RANKED = ("assign", "status", "domain", "score", "alt_node", "alt_score")


def need_free(nbytes: int, what: str) -> None:
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip(f"{what}: needs {nbytes / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free")


def engine(topo, chunk: int, lvl=None):
    from gpu_util import new_engine
    eng = new_engine(topo, chunk_nodes=chunk)
    if lvl is not None:
        eng.set_exclusive_levels(lvl[1:], np.zeros((0, 3), np.int32))
    return eng


def bits_equal(got, exp, tag):
    g = np.ascontiguousarray(got)
    e = np.ascontiguousarray(exp)
    if g.dtype.kind == "f":
        g, e = g.view(np.uint32), e.view(np.uint32)
    assert g.shape == e.shape, (tag, g.shape, e.shape)
    bad = np.argwhere(g != e)
    assert len(bad) == 0, (tag, f"{len(bad)} differ, first at {tuple(int(v) for v in bad[0])}", g[tuple(bad[0])],
                           e[tuple(bad[0])])


def check_ranked(got, exp: wm.Expect, tag, n=6):
    for name, x in zip(RANKED[:n], got):
        bits_equal(x, getattr(exp, name), (tag, name))


@pytest.fixture(scope="module")
def fleet():
    return wm.groups_fleet()


@pytest.fixture(scope="module")
def fleet_ref(fleet):
    per, rows, topk = wm.groups_oracle(fleet)
    return wm.expand(fleet, per, wm.replica_spans(fleet)), rows, topk


def check_rows(eng, h, fleet, rows, topk, tag):
    """Every row of the handle against its group's and role's oracle row, and the top-K keys of every role row."""
    for g in range(len(fleet.groups)):
        want, keys = rows[(fleet.rep[g], 0)], topk[(fleet.rep[g], 0)]
        for p in range(wm.Q):
            r = wm.Q * g + p
            got = eng.read_scores(h, r)
            if not np.array_equal(got.view(np.uint32), want[p].view(np.uint32)):
                bad = np.nonzero(got.view(np.uint32) != want[p].view(np.uint32))[0]
                raise AssertionError(f"{tag}: row {r} (group {g}, role {p}): {len(bad)} nodes differ, first {bad[0]}, "
                                     f"last {bad[-1]}: gpu={got[bad[0]]} oracle={want[p][bad[0]]}")
            assert np.array_equal(eng.read_topk(h, r, 32), keys[p]), (tag, "topk", g, p)


def staged_groups(eng, fleet, ref, tag):
    exp, rows, topk = ref
    h = eng.stage_groups(fleet.blob)
    try:
        eng.run_staged(h, 1)
        a, s, d = eng.fetch(h)
        check_ranked((a, s, d), exp, tag, 3)
        tm = eng.last_timing()
        check_rows(eng, h, fleet, rows, topk, tag)
    finally:
        eng.release(h)
    n = fleet.topo.n
    words = int(plan_steps(fleet.blob, n, len(fleet.topo.domain_owner))[:, 3].max())
    assert tm["scores"] == ROWS * n > 1 << 31, (tag, tm["scores"])
    assert tm["algo_bytes"] == 4 * ROWS * n + 4 * words + 8 * n > 1 << 32, (tag, tm["algo_bytes"])


@pytest.mark.parametrize("chunk", wm.CHUNKS, ids=CHUNK_IDS)
def test_groups_fleet(fleet, fleet_ref, chunk):
    """stage_groups + run_staged + fetch + every row, place_groups (direct) and place_groups_ranked with n_alt 8."""
    need_free(wm.need_bytes(ROWS, wm.N, chunk), "groups fleet")
    exp = fleet_ref[0]
    eng = engine(fleet.topo, chunk)
    try:
        staged_groups(eng, fleet, fleet_ref, f"staged/{chunk}")
        check_ranked(eng.place_groups(fleet.blob), exp, f"direct/{chunk}", 3)
        if not any(os.environ.get(v) for v in SWITCHES_OFF_DIRECT):   # the direct path's own counters
            tm = eng.last_timing()
            assert tm["algo_bytes"] == 4 * ROWS * wm.N + 4 * len(fleet.blob) + 8 * wm.N, tm
            assert tm["scores"] == ROWS * wm.N, tm
        check_ranked(eng.place_groups_ranked(fleet.blob, 8), exp, f"ranked/{chunk}")
    finally:
        eng.close()


def test_reuse_wide_small_wide(fleet, fleet_ref):
    """One context: the wide plan, a three-group plan in the same buffers, the wide plan again."""
    need_free(wm.need_bytes(ROWS, wm.N), "reuse")
    exp, rows, topk = fleet_ref
    small = wm.Fleet(fleet.topo, [fleet.groups[g] for g in (0, 1, 891)], None, [0, 1, 2], [0, 1, 2], fleet.pivots,
                     {})
    small.blob = wm._build(small.groups)
    eng = engine(fleet.topo, 0)
    try:
        staged_groups(eng, fleet, fleet_ref, "wide 1")
        got = eng.place_groups_ranked(small.blob, 8)
        for k, g in enumerate((0, 1, 891)):
            sl = slice(wm.Q * g, wm.Q * (g + 1))
            for name, x in zip(RANKED, got):
                y = getattr(exp, name)
                bits_equal(x[wm.Q * k:wm.Q * (k + 1)] if name not in ("status", "domain") else x[k],
                           y[sl] if name not in ("status", "domain") else y[g], ("small", name, g))
        h = eng.stage_groups(small.blob)
        try:
            eng.run_staged(h, 1)
            for k, g in enumerate((0, 1, 891)):
                for p in range(wm.Q):
                    bits_equal(eng.read_scores(h, wm.Q * k + p), rows[(fleet.rep[g], 0)][p], ("small row", g, p))
        finally:
            eng.release(h)
        staged_groups(eng, fleet, fleet_ref, "wide 2")
        check_ranked(eng.place_groups_ranked(fleet.blob, 8), exp, "wide 2 ranked")
    finally:
        eng.close()


@pytest.fixture(scope="module")
def steps():
    sf = wm.steps_fleet()
    return sf, wm.steps_oracle(sf)


@pytest.mark.parametrize("chunk", wm.CHUNKS, ids=CHUNK_IDS)
def test_step_batch(steps, chunk):
    """stage + run_staged + every row + read_topk, and score_assign.  The straddling steps are hub-anchored: their
    rows are read back through k_select_assign's global candidate list."""
    sf, per = steps
    need_free(wm.need_bytes(ROWS, wm.N, chunk), "step batch")
    ns = len(sf.steps)
    exp_a = np.concatenate([per[sf.rep[s]]["assign"] for s in range(ns)])
    exp_s = np.concatenate([per[sf.rep[s]]["status"] for s in range(ns)])
    exp_d = np.concatenate([per[sf.rep[s]]["domain"] for s in range(ns)])
    eng = engine(sf.topo, chunk)
    try:
        h = eng.stage(sf.blob)
        try:
            eng.run_staged(h, 1)
            a, s, d = eng.fetch(h)
            bits_equal(a, exp_a, "assign")
            bits_equal(s, exp_s, "status")
            bits_equal(d, exp_d, "domain")
            tm = eng.last_timing()
            for st in range(ns):
                ref = per[sf.rep[st]]
                for p in range(wm.Q):
                    r = wm.Q * st + p
                    bits_equal(eng.read_scores(h, r), ref["matrix"][p], ("row", chunk, st, p))
                    assert np.array_equal(eng.read_topk(h, r, 32), ref["topk"][p]), ("topk", chunk, st, p)
        finally:
            eng.release(h)
        assert tm["scores"] == ROWS * wm.N > 1 << 31, tm
        assert tm["algo_bytes"] == 4 * ROWS * wm.N + 4 * len(sf.blob) + 8 * wm.N > 1 << 32, tm
        a2, s2, d2 = eng.score_assign(sf.blob)
        bits_equal(a2, exp_a, "score_assign")
        bits_equal(s2, exp_s, "score_assign status")
        bits_equal(d2, exp_d, "score_assign domain")
    finally:
        eng.close()


@pytest.fixture(scope="module")
def lw_case(fleet):
    rp = wm.lw_role_pods(fleet)
    return rp, wm.expand(fleet, wm.lw_oracle(fleet, rp), wm.lw_spans(fleet, rp))


@pytest.mark.parametrize("chunk", wm.CHUNKS, ids=CHUNK_IDS)
def test_leader_worker(fleet, lw_case, chunk):
    """place_groups_lw and place_groups_lw_ranked (n_alt 8, kept rows past 2^31 floats), S in {1, 2, 4} and C in
    {-1, 0, 1} on the straddle groups."""
    rp, exp = lw_case
    need_free(wm.need_bytes(ROWS, wm.N, chunk, copies=2), "leader-worker")
    eng = engine(wm.lw_topology(fleet.topo), chunk, wm.lw_levels(fleet.topo))
    try:
        check_ranked(eng.place_groups_lw(fleet.blob, rp), exp, f"lw/{chunk}", 3)
        check_ranked(eng.place_groups_lw_ranked(fleet.blob, rp, 8), exp, f"lw ranked/{chunk}")
    finally:
        eng.close()


@pytest.fixture(scope="module")
def rerun(fleet):
    rf = wm.rerun_fleet(topo=fleet.topo)
    per, _, _ = wm.groups_oracle(rf)
    return rf, wm.expand(rf, per, wm.replica_spans(rf))


@pytest.mark.parametrize("chunk", wm.CHUNKS, ids=CHUNK_IDS)
def test_rerun_fleet_ranked(rerun, chunk):
    """Every group re-run by the host-driven loop: place_groups_ranked keeps the first wave's 7 200 rows in b->kept,
    then the second wave's 900 from past 2^31 floats, and ranks the alternates from them."""
    rf, exp = rerun
    assert (exp.status == 1).all()
    need_free(wm.need_bytes(ROWS + wm.G, wm.N, chunk, copies=2), "re-run fleet")
    eng = engine(rf.topo, chunk)
    try:
        check_ranked(eng.place_groups_ranked(rf.blob, 8), exp, f"rerun/{chunk}")
        check_ranked(eng.place_groups(rf.blob), exp, f"rerun unranked/{chunk}", 3)
    finally:
        eng.close()


def test_per_wave_selection_past_shared_memory():
    """Groups 890 and 891, which hold r* of both configurations, carry 2 000 more scheduled pods on distinct nodes: the
    plan does not fit k_plan_group, so it runs one launch per wave and k_select_assign corrects and reads the rows."""
    need_free(wm.need_bytes(ROWS, wm.N), "per-wave plan")
    f = wm.groups_fleet(heavy=(890, 891))
    per, rows, topk = wm.groups_oracle(f)
    ref = (wm.expand(f, per, wm.replica_spans(f)), rows, topk)
    for chunk in wm.CHUNKS:
        eng = engine(f.topo, chunk)
        try:
            staged_groups(eng, f, ref, f"per-wave/{chunk}")
            assert eng.stats()["plan_ctas"] == 0
            check_ranked(eng.place_groups(f.blob), ref[0], f"per-wave direct/{chunk}", 3)
            check_ranked(eng.place_groups_ranked(f.blob, 8), ref[0], f"per-wave ranked/{chunk}")
        finally:
            eng.close()


# ---- the node ceiling: N = 1 638 400, 170 groups

CEIL_N, CEIL_G = 1_638_400, 170


def test_node_ceiling():
    """rbgtopo's node ceiling: 1 360 role rows pass 2^31 floats.  place_groups_ranked and place_groups_lw_ranked."""
    r, nstar = wm.straddle(CEIL_N)
    assert CEIL_G * wm.Q > r and (r, nstar) == (1310, 1_179_648)
    need_free(wm.need_bytes(CEIL_G * wm.Q, CEIL_N, copies=2), "node ceiling")
    g = r // wm.Q
    f = wm.groups_fleet(CEIL_N, CEIL_G, (g - 1, g, g + 1), piv=[nstar])
    per, _, _ = wm.groups_oracle(f)
    exp = wm.expand(f, per, wm.replica_spans(f))
    rp = wm.lw_role_pods(f)
    lexp = wm.expand(f, wm.lw_oracle(f, rp), wm.lw_spans(f, rp))
    eng = engine(f.topo, 0)
    try:
        check_ranked(eng.place_groups_ranked(f.blob, 8), exp, "ceiling ranked")
    finally:
        eng.close()
    eng = engine(wm.lw_topology(f.topo), 0, wm.lw_levels(f.topo))
    try:
        check_ranked(eng.place_groups_lw_ranked(f.blob, rp, 8), lexp, "ceiling lw ranked")
    finally:
        eng.close()


# ---- library switches, read when the library loads

@pytest.mark.parametrize("var", ["RBGTOPO_NO_DIRECT", "RBGTOPO_PER_WAVE_PLAN", "RBGTOPO_SPLIT_MIN_GROUPS=2",
                                 "RBGTOPO_CONCURRENT_PLAN", "RBGTOPO_EMIT_ROWS=1", "RBGTOPO_EMIT_ROWS=12"])
def test_switches_in_a_subprocess(var):
    """RBGTOPO_NO_DIRECT: place_groups through the staged path; RBGTOPO_PER_WAVE_PLAN: one launch per wave;
    RBGTOPO_SPLIT_MIN_GROUPS=2: place_groups as two halves; RBGTOPO_CONCURRENT_PLAN: k_plan_correct writes the
    corrections; RBGTOPO_EMIT_ROWS=1 / 12: k_emit_rows segments of 1 / 12 rows instead of 6, which move the segment
    boundaries relative to r*.  Each runs the groups fleet in both chunk configurations."""
    need_free(wm.need_bytes(ROWS, wm.N), var)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ)
    name, _, val = var.partition("=")
    env[name] = val or "1"
    r = subprocess.run([sys.executable, "-m", "pytest", "tests/test_gpu_wide_matrix.py", "-q", "-m", "gpu", "-x",
                        "-p", "no:cacheprovider", "-k", "test_groups_fleet"],
                       cwd=root, env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert "2 passed" in r.stdout, r.stdout[-2000:]
