"""GPU: committed leader-worker batches at exclusive levels at their limits (rbgtopo_place_groups_lw_committed[_ranked]
on a ctx with RBGTOPO_CFG_LW_COMMIT_LEVELS, DESIGN.md §3.16) bit for bit against tests/lw_committed_levels_oracle.py on
the cases of tests/lw_commit_levels_limits_cases.py: assign, status, domain, the replayed round count where the case
pins it, the ranked call at n_alt 0, 1 and 8 (all seven outputs, fp32 as bits) and the invariants read from the outputs
alone.  Also: one mixed-level wave under every emit block size, 128-node chunks with a one-node tail, uploads that do
not grow with the claimed domains, refreshes during a ~100-round call, the §3.11 exactness bound at a level, and the
scale cases (2^20 + 1 nodes at seven levels, the room bitmap's 1 638 400 nodes)."""
import json
import os
import resource
import subprocess
import sys
import threading
import time

import numpy as np
import pytest

import lw_commit_levels_limits_cases as lc
from rbg_b200 import synth
from rbg_b200.engine import TopoPlacer
from test_gpu_lw_committed_alternates import bits
from test_oracle_lw_committed_levels_limits import invariants

pytestmark = pytest.mark.gpu

CASES = lc.cases()
HERE = os.path.dirname(os.path.abspath(__file__))


def engine(c, **kw):
    eng = TopoPlacer(device=0, lw_committed_levels=True, **kw)
    t = c.topo
    eng.set_topology(t.row_ptr, t.col_idx, t.edge_w, t.free, t.domain, t.domain_owner)
    eng.set_exclusive_levels(c.lv[1:], c.occ, level_n_domains=c.nd[1:])
    return eng


def same(x, y):
    return all(np.array_equal(np.asarray(p), np.asarray(q)) for p, q in zip(x[:3], y[:3]))


def check(eng, c, brute_force=True, exp=None):
    got = eng.place_groups_lw_committed(c.blob(), c.role_pods())
    a, s, d, rounds = got
    ea, es, ed = c.expected() if exp is None else exp
    assert np.array_equal(a, ea), (c.name, np.nonzero(a != ea)[0][:8])
    assert np.array_equal(s, es) and np.array_equal(d, ed), (c.name, s, es, d, ed)
    if c.rounds is not None:
        assert rounds == c.rounds, (c.name, rounds, c.rounds)
    else:
        assert 1 <= rounds <= len(c.groups), (c.name, rounds)
    if brute_force:
        invariants(c, a, s, d)
    return got


def check_ranked(eng, c, got, exp=None):
    exp = c.expected_ranked(8) if exp is None else exp
    for F in (0, 1, 8):
        r = eng.place_groups_lw_committed_ranked(c.blob(), c.role_pods(), F)
        assert same(r, got) and r[3] == got[3], (c.name, F)
        sc, an, asc = (np.asarray(x) for x in r[4:])
        assert np.array_equal(bits(sc), bits(exp[3])), (c.name, F, np.nonzero(bits(sc) != bits(exp[3]))[0][:8])
        assert an.size == asc.size == F * len(sc), (c.name, F)
        assert np.array_equal(an.reshape(len(sc), F), exp[4][:, :F]), (c.name, F)
        assert np.array_equal(bits(asc).reshape(len(sc), F), bits(exp[5][:, :F])), (c.name, F)


@pytest.mark.parametrize("i", range(len(CASES)), ids=[c.name for c in CASES])
def test_cases_match_the_oracle_plain_and_ranked(i):
    c = CASES[i]
    eng = engine(c)
    try:
        check_ranked(eng, c, check(eng, c))
    finally:
        eng.close()


# ---- one mixed-level wave under every emit block size (read once, when the library loads)
_EMIT_SCRIPT = """
import sys, json
import numpy as np
sys.path[:0] = [{root!r}, {tests!r}]
import lw_commit_levels_limits_cases as lc
from test_gpu_lw_committed_levels_limits import engine
c = lc.emit_blocks()
eng = engine(c)
r = eng.place_groups_lw_committed(c.blob(), c.role_pods())
k = eng.place_groups_lw_committed_ranked(c.blob(), c.role_pods(), 8)
eng.close()
print(json.dumps([np.asarray(x).view(np.int32).tolist() if hasattr(x, "view") else x for x in list(r) + list(k)]))
"""


def test_emit_block_sizes_agree_on_a_mixed_level_wave():
    c = lc.emit_blocks()
    out = {}
    for blk in ("1", None, "16"):
        env = {k: v for k, v in os.environ.items() if k != "RBGTOPO_EMIT_BLOCK"}
        if blk is not None:
            env["RBGTOPO_EMIT_BLOCK"] = blk
        p = subprocess.run([sys.executable, "-c", _EMIT_SCRIPT.format(root=os.path.dirname(HERE), tests=HERE)],
                           env=env, capture_output=True, text=True, timeout=600)
        assert p.returncode == 0, p.stderr[-2000:]
        out[blk] = json.loads(p.stdout.strip().splitlines()[-1])
    assert out["1"] == out[None] == out["16"]
    ea, es, ed = c.expected()
    r = out[None]
    assert r[0] == ea.tolist() and r[1] == es.tolist() and r[2] == ed.tolist()
    exp = c.expected_ranked(8)
    assert r[4:7] == r[0:3] and r[7] == r[3]
    i32 = lambda x: bits(x).view(np.int32).ravel().tolist()
    flat = lambda x: np.asarray(x).ravel().tolist()
    assert flat(r[8]) == i32(exp[3]) and flat(r[9]) == flat(exp[4]) and flat(r[10]) == i32(exp[5])


@pytest.mark.parametrize("n", [4097, 129])
def test_ragged_chunks_of_128_nodes(n):
    """chunk_nodes = 128: N = 4 097 is 33 chunks with a one-node tail; the best node is the last."""
    c = lc.ragged(n)
    for kw in (dict(chunk_nodes=128), {}):
        eng = engine(c, **kw)
        try:
            check_ranked(eng, c, check(eng, c))
        finally:
            eng.close()


# ---- uploads grow with groups and pods, not with the claimed domains
def padded(c, k: int):
    """c with k isolated free-0 nodes appended per node, in that node's domain at every level: every claimed domain
    grows (k + 1) times, nothing else changes."""
    n = c.topo.n
    src = np.concatenate([np.arange(n), np.repeat(np.arange(n), k)])
    m = len(src)
    row_ptr = np.concatenate([c.topo.row_ptr, np.full(m - n, c.topo.row_ptr[-1], np.int32)]).astype(np.int32)
    free = np.concatenate([c.topo.free, np.zeros(m - n, np.int32)]).astype(np.int32)
    lv = c.lv[:, src].astype(np.int32)
    topo = synth.Topology(row_ptr, c.topo.col_idx, c.topo.edge_w, free, lv[0].copy(), c.topo.domain_owner.copy())
    return c.replace(topo=topo, lv=lv)


def test_uploads_do_not_grow_with_the_claimed_domains():
    base = lc.churn("shrink")
    small, big = padded(base, 3), padded(base, 63)
    sizes = lambda x: np.bincount(x.lv[2])
    assert (sizes(big) == 16 * sizes(small)).all()
    es, eb = small.expected(), big.expected()
    assert same(es, eb) and len(lc.replay(small)) == len(lc.replay(big)) == 3
    out = []
    for c in (small, big):
        eng = engine(c)
        try:
            got = check(eng, c)
            t = eng.last_timing()
            out.append((got[3], t["h2d_words"], t["launches"]))
        finally:
            eng.close()
    assert out[0] == out[1], out


# ---- refreshes issued while a ~100-round call runs
def _refreshed(c, kind):
    a0 = c.extra["a"][0]
    if kind == "free":
        free = c.topo.free.copy()
        free[a0] = 0
        t = synth.Topology(c.topo.row_ptr, c.topo.col_idx, c.topo.edge_w, free, c.topo.domain, c.topo.domain_owner)
        return (lambda e: e.update_nodes(free=free)), c.replace(topo=t)
    if kind == "records":
        occ = np.array([[a0, 99, 1]], np.int32)
        return (lambda e: e.set_exclusive_levels(None, occ)), c.replace(occ=occ)
    lv = np.stack([c.lv[0]] + [np.arange(c.topo.n)] * 7).astype(np.int32)
    nd = [c.nd[0]] + [c.topo.n] * 7
    return (lambda e: e.set_exclusive_levels(lv[1:], c.occ, level_n_domains=nd[1:])), c.replace(lv=lv, nd=nd)


@pytest.mark.parametrize("kind", ["free", "records", "partitions"])
def test_a_refresh_during_a_call_lands_between_calls(kind, record_property):
    c = lc.chain(*lc.REFRESH_CHAIN)
    refresh, new_c = _refreshed(c, kind)
    old, new = c.expected(), new_c.expected()
    assert not same(old, new)
    eng = engine(c)
    try:
        out = {}
        started = threading.Event()

        def call():
            started.set()
            t0 = time.perf_counter()
            out["r"] = eng.place_groups_lw_committed(c.blob(), c.role_pods())
            out["call"] = (t0, time.perf_counter())
        t = threading.Thread(target=call)
        t.start()
        started.wait()
        time.sleep(0.002)
        r0 = time.perf_counter()
        refresh(eng)
        t.join()
        r = out["r"]
        assert same(r, old) != same(r, new), "a result mixed of two snapshots"
        c0, c1 = out["call"]
        record_property("snapshot_seen", "old" if same(r, old) else "new")
        record_property("call_ms", round(1e3 * (c1 - c0), 3))
        record_property("refresh_issued_ms", round(1e3 * (r0 - c0), 3))
        if same(r, old):
            assert r[3] == lc.REFRESH_CHAIN[0]
        assert same(eng.place_groups_lw_committed(c.blob(), c.role_pods()), new)
    finally:
        eng.close()


# ---- the exactness bound with the group at a level
@pytest.mark.parametrize("case_i", range(5))
def test_exactness_bound_at_a_level(case_i):
    """test_gpu_lw_limits.EXACT_CASES with the group exclusive at level 2 (its real roles participating) on a
    flags = 7 ctx: at the bound both committed calls return RBGTOPO_EINEXACT and leave their sentinel outputs
    untouched; one anchor below they place like the oracle, through the level view and the claim lists."""
    from test_gpu_lw_committed_alternates import raw, untouched as all_sentinel
    from test_gpu_lw_limits import raw as raw_plain
    at, c_at = lc.exact(case_i)
    eng = engine(at(0))
    try:
        c = at(c_at)
        gb, rp = c.blob(), c.role_pods()
        rc, untouched = raw_plain(eng, "lw_committed", gb, rp)
        assert rc == -4 and untouched, ("plain", rc, c_at)
        rc, out = raw(eng, gb, rp, 8)
        assert rc == -4 and all_sentinel(out), ("ranked", rc, c_at)
        c = at(c_at - 1)
        check_ranked(eng, c, check(eng, c))
    finally:
        eng.close()


# ---- scale
@pytest.mark.parametrize("which", ["million", "bitmap_ceiling"])
def test_scale(which, capsys):
    """2^20 + 1 nodes with seven levels, 610 000 records and 12 groups (lc.million), and the room bitmap's 1 638 400
    nodes with three levels (every group places; one node more is refused elsewhere).  Prints the wall time of the
    case (build, oracle, install and call) and the peak host RSS of the test process up to the end of the case
    (ru_maxrss: the largest of everything the session ran so far, not the case's own).  The brute-force anti-affinity
    check over every record is skipped here: the bit-for-bit oracle comparison stands for it."""
    t0 = time.perf_counter()
    c = getattr(lc, which)()
    exp = c.expected()
    assert (exp[1] != 2).any()
    eng = engine(c)
    try:
        got = check(eng, c, brute_force=False, exp=exp)
        if which == "bitmap_ceiling":
            assert (got[1] == 0).all()
    finally:
        eng.close()
    wall = time.perf_counter() - t0
    rss = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1024
    with capsys.disabled():
        print(f"\n{c.name}: N {c.topo.n}, levels {c.lv.shape[0] - 1}, groups {len(c.groups)}, rounds {got[3]}, "
              f"wall {wall:.1f} s (build, oracle, install and call), peak host RSS of the process so far {rss:.0f} MiB")
