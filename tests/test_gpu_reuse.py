"""GPU, one device: pooled batch reuse.

Every entry point runs on a batch of the context's pool, and one caller always gets the pool's first free batch: the
calls of a scheduler run one after another on the same device and pinned buffers, which only grow and are never
cleared, and on per-batch flags each path resets on its own.  Here every call B runs on a context that has just run
some other call A, and B's outputs (float outputs as bits), the dense rows and top-K lists a staged pass defines and
the call's counters (launches, h2d_words, scores, algo_bytes) must equal those of B on a fresh context with the same
snapshot, partitions and refresh history.  The fresh result is checked once per (B, fixture) against the oracle.

Cases: every entry point (tests/reuse_cases.py KINDS) with the large fixture before B with the small one and the other
way round, on a level-0 context and on the flags = 7 context with levels installed, and on the split and staged paths
of place_groups in a subprocess; calls that fail after their blob was uploaded (EINVAL late in a large blob, ELIMIT,
EINEXACT at the exactness bounds); a context whose topology changes size under its pool; a world = 2 pair of contexts
on one device; a seeded sequence with refreshes, held staged handles and the timed path; threads sharing one
context."""
import functools
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

import groups_gen as gg
import reuse_cases as rc
from gpu_util import check_batch
from rbg_b200 import synth
from rbg_b200.engine import RbgTopoError, TopoPlacer, plan_steps

pytestmark = pytest.mark.gpu

COUNTERS = ("launches", "h2d_words", "scores", "algo_bytes")
NAMES = {"score_assign": ("assign", "status", "domain"),
         "direct": ("assign", "status", "domain"),
         "committed": ("assign", "status", "domain", "rounds"),
         "lw": ("assign", "status", "domain"),
         "lw_committed": ("assign", "status", "domain", "rounds"),
         "ranked": ("assign", "status", "domain", "score", "alt_node", "alt_score"),
         "lw_ranked": ("assign", "status", "domain", "score", "alt_node", "alt_score"),
         "committed_ranked": ("assign", "status", "domain", "rounds", "score", "alt_node", "alt_score"),
         "lw_committed_ranked": ("assign", "status", "domain", "rounds", "score", "alt_node", "alt_score")}


@functools.lru_cache(maxsize=None)
def world(name):
    if name == "plain":
        return rc.plain_world()
    if name == "levels":
        return rc.level_world()
    if name == "level0":
        return rc.level0_world()
    return rc.plain_world(seed=rc.TOPO_SEED, n=int(name[4:]))   # "topoN": a world of the topology-change sequence


def make_engine(w, refreshes=(), timing=False, rank=0, n_ranks=1):
    eng = TopoPlacer(device=0, rank=rank, world=n_ranks, **w.flags)
    t = w.topo
    eng.set_topology(t.row_ptr, t.col_idx, t.edge_w, t.free, t.domain, t.domain_owner)
    if w.lv is not None:
        eng.set_exclusive_levels(w.lv[1:], w.occ, level_n_domains=w.nd[1:])
    for r in refreshes:
        r(eng)
    if timing:
        eng.set_kernel_timing(True)
    return eng


def _bits(x):
    x = np.ascontiguousarray(x)
    return x.view(np.uint32) if x.dtype == np.float32 else x


def defined_rows(w, fx, assign):
    """The replica rows and role rows of a staged GROUPS pass whose content it defines: every wave of a group up to and
    including the first wave in which the group lost a replica (later waves are not selected; their rows hold
    whatever the buffers held).  tests/test_gpu_groups_limits.defined_rows, from the fetched placements."""
    first = {(int(s[0]), int(s[1])): (int(s[4]), int(s[5]))
             for s in plan_steps(fx.blob, w.topo.n, len(w.topo.domain_owner))}
    rows, roles, off = [], [], 0
    for gi, g in enumerate(fx.groups):
        start = np.concatenate([[0], np.cumsum([r[1] for r in g.roles])])
        for wi, wave in enumerate(gg.waves_of(g.roles)):
            row0, role0 = first[(gi, wi)]
            rows += range(row0, row0 + sum(t for _, _, t in wave))
            roles += range(role0, role0 + len(wave))
            idx = [off + int(start[ri]) + f + j for ri, f, t in wave for j in range(t)]
            if (assign[idx] < 0).any():
                break
        off += int(start[-1])
    return rows, roles


def staged_result(eng, w, fx, h):
    """fetch, then every dense row and top-K list the last pass of handle h defines."""
    a, s, d = eng.fetch(h)
    if fx.family == "steps":
        rows, roles = range(int(fx.blob[4])), range(int(fx.blob[5]))
    else:
        rows, roles = defined_rows(w, fx, a)
    m = np.stack([eng.read_scores(h, r).view(np.uint32) for r in rows]) if len(rows) else np.zeros((0, 0), np.uint32)
    topk = np.stack([eng.read_topk(h, p, 32) for p in roles]) if len(roles) else np.zeros((0, 32), np.uint64)
    return {"assign": a.copy(), "status": s.copy(), "domain": d.copy(), "rows": m, "topk": topk,
            "row_ids": np.asarray(rows, np.int64)}


def run(kind, eng, w, fx, counters=True):
    """One call of `kind` on fx; its outputs by name, and the call's counters."""
    if kind in ("steps", "staged"):
        h = eng.stage(fx.blob) if kind == "steps" else eng.stage_groups(fx.blob)
        try:
            eng.run_staged(h, 1)
            out = staged_result(eng, w, fx, h)
            t = eng.last_timing() if counters else {}
        finally:
            eng.release(h)
    else:
        f = {"score_assign": lambda: eng.score_assign(fx.blob),
             "direct": lambda: eng.place_groups(fx.blob),
             "committed": lambda: eng.place_groups_committed(fx.blob),
             "committed_ranked": lambda: eng.place_groups_committed_ranked(fx.blob, rc.N_ALT),
             "ranked": lambda: eng.place_groups_ranked(fx.blob, rc.N_ALT),
             "lw": lambda: eng.place_groups_lw(fx.blob, fx.rp),
             "lw_ranked": lambda: eng.place_groups_lw_ranked(fx.blob, fx.rp, rc.N_ALT),
             "lw_committed": lambda: eng.place_groups_lw_committed(fx.blob, fx.rp),
             "lw_committed_ranked": lambda: eng.place_groups_lw_committed_ranked(fx.blob, fx.rp, rc.N_ALT)}[kind]
        out = {n: np.array(x, copy=True) for n, x in zip(NAMES[kind], f())}
        t = eng.last_timing() if counters else {}
    for c in COUNTERS if counters else ():
        out["t_" + c] = np.asarray(t[c])
    return out


def same(got, exp, tag):
    """Bit equality of two run() results (the counters only where both have them), naming the first difference."""
    for name, y in exp.items():
        if name not in got:
            assert name.startswith("t_"), (tag, name)
            continue
        x, y = np.atleast_1d(got[name]), np.atleast_1d(y)   # the counters are scalars
        assert x.shape == y.shape, (tag, name, x.shape, y.shape)
        bad = np.argwhere(_bits(x) != _bits(y))
        assert len(bad) == 0, (tag, name, f"{len(bad)} differ, first at {tuple(int(v) for v in bad[0])}",
                               x[tuple(bad[0])], y[tuple(bad[0])])


# ---- the oracle, once per (world, kind, fixture), on the fresh context

def _oracle_topo(w):
    t = w.topo
    return synth.Topology(t.row_ptr, t.col_idx, t.edge_w, t.free, t.domain, np.asarray(w.owner0(), np.int32))


def oracle_check(kind, eng, w, fx, got):
    import test_gpu_alternates as ta
    import test_gpu_committed as tc
    import test_gpu_committed_alternates as tca
    import test_gpu_lw as tl
    import test_gpu_lw_alternates as tla
    import test_gpu_lw_committed as tlc
    import test_gpu_lw_committed_alternates as tlca
    import test_gpu_lw_committed_levels as tlcl
    import lw_commit_levels_gen as lvg
    from test_gpu_groups_limits import check_direct, check_staged, oracle_plan
    from test_gpu_groups_limits import defined_rows as oracle_rows
    topo = w.topo
    if kind in ("score_assign", "steps"):
        check_batch(eng, _oracle_topo(w), fx.blob)
        return
    if w.lv is not None:
        # at levels >= 1 the oracle with a helper for such fleets is that of committed leader-worker batches; with one pod
        # per replica it is place_groups_committed's, and on one group at a time place_groups' and place_groups_lw's
        # (test_gpu_lw_committed_levels: test_one_pod_per_replica_is_place_groups_committed,
        # test_one_group_batches_are_place_groups_lw)
        f = lvg.LvFleet(topo, fx.groups, [[tuple(int(v) for v in x) for x in fx.rp]] if fx.rp is not None else [],
                        w.lv, w.nd, w.occ)
        ones = [[(1, -1)] * len(g.roles) for g in fx.groups]
        if kind in ("committed", "direct", "lw"):
            if kind == "committed":
                exp = lvg.LvFleet(topo, fx.groups, ones, w.lv, w.nd, w.occ).expected()
            else:
                rps = ones
                if kind == "lw":
                    cut = np.cumsum([0] + [len(g.roles) for g in fx.groups])
                    rps = [[tuple(int(v) for v in x) for x in fx.rp[cut[k]:cut[k + 1]]] for k in range(len(fx.groups))]
                one = [lvg.LvFleet(topo, [g], [rp], w.lv, w.nd, w.occ).expected() for g, rp in zip(fx.groups, rps)]
                exp = [np.concatenate([np.asarray(e[i]) for e in one]) for i in range(3)]
            same({k: got[k] for k in ("assign", "status", "domain")},
                 dict(zip(("assign", "status", "domain"), (np.asarray(x, np.int32) for x in exp))), ("oracle", kind))
        elif kind == "lw_committed":
            tlcl.check(eng, f)
        elif kind == "lw_committed_ranked":
            exp = f.expected_ranked(rc.N_ALT)
            same({k: got[k] for k in NAMES[kind] if k != "rounds"},
                 dict(zip(("assign", "status", "domain", "score", "alt_node", "alt_score"), exp)), "oracle")
        return
    gb, rp = fx.blob, fx.rp
    if kind in ("direct", "staged"):
        states, waves = oracle_plan(topo, gb)
        if kind == "direct":
            check_direct(eng, states, gb)
        else:
            check_staged(eng, topo, states, waves, gb)
            rows, roles = oracle_rows(topo, states, waves, gb)
            assert sorted(got["row_ids"].tolist()) == sorted(rows), "defined rows"   # ours group-major, its wave-major
    elif kind == "committed":
        tc.check(eng, topo, gb, fast=True)
    elif kind == "committed_ranked":
        tca.check(eng, topo, gb, rc.N_ALT)
    elif kind == "ranked":
        ta.check(eng, topo, gb, rc.N_ALT)
    elif kind == "lw":
        tl.check(eng, topo, gb, rp)
    elif kind == "lw_ranked":
        tla.check(eng, topo, gb, rp, rc.N_ALT)
    elif kind == "lw_committed":
        tlc.check(eng, topo, gb, rp)
    elif kind == "lw_committed_ranked":
        tlca.check(eng, topo, gb, rp, n_alts=(rc.N_ALT,))


ORACLE_WORLDS = ("plain", "levels", "topo129", "topo4097")
_EXP = {}


def expected(wname, kind, size, version=0, refreshes=(), timing=False, fx=None, rank=0, n_ranks=1):
    """kind on a FRESH context of the world after `refreshes` (snapshot `version`); the oracle checks the first one
    (one rank of n_ranks > 1: test_world2_pair_of_contexts compares its placements with one rank's)."""
    key = (wname, kind, size, version, timing, rank, n_ranks)
    if key not in _EXP:
        w = world(wname)
        fx = fx or w.fixture(kind, size)
        eng = make_engine(w, refreshes, timing, rank, n_ranks)
        try:
            _EXP[key] = run(kind, eng, w, fx)
            if version == 0 and not timing and n_ranks == 1 and wname in ORACLE_WORLDS:
                oracle_check(kind, eng, w, fx, _EXP[key])
        finally:
            eng.close()
    return _EXP[key]


def run_checked(eng, wname, kind, size, tag, **kw):
    w = world(wname)
    same(run(kind, eng, w, w.fixture(kind, size)), expected(wname, kind, size, **kw), tag)


# ---- 1. every ordered pair

@pytest.mark.parametrize("wname", ["plain", "levels"])
def test_every_ordered_pair(wname):
    """For every (A, B) in K x K on one context: A large then B small, A small then B large; every call against its
    fresh-context result."""
    eng = make_engine(world(wname))
    try:
        for a in rc.KINDS:
            for b in rc.KINDS:
                for sa, sb in (("large", "small"), ("small", "large")):
                    run_checked(eng, wname, a, sa, (wname, "A", a, sa, "B", b, sb))
                    run_checked(eng, wname, b, sb, (wname, "B", b, sb, "after", a, sa))
    finally:
        eng.close()


@pytest.mark.parametrize("var", ["RBGTOPO_SPLIT_MIN_GROUPS", "RBGTOPO_NO_DIRECT"])
def test_every_ordered_pair_on_other_paths_in_a_subprocess(var):
    """RBGTOPO_SPLIT_MIN_GROUPS=1: place_groups pipelines the fleet as two halves on two batches of the pool;
    RBGTOPO_NO_DIRECT: place_groups through the staged path (expanded plan, early emit)."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ)
    env[var] = "1"
    r = subprocess.run([sys.executable, "-m", "pytest", "tests/test_gpu_reuse.py", "-q", "-m", "gpu", "-x",
                        "-k", "test_every_ordered_pair and not subprocess"], cwd=root, env=env, capture_output=True,
                       text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert "2 passed" in r.stdout, r.stdout[-2000:]


@pytest.mark.parametrize("b", ["fits", "grows"])
def test_growth_rule_either_side(b):
    """A: one 8-role step (the dense matrix reserved for grow(8 rows)); B: 10 role rows, inside that capacity with
    A's stale tail, or 11, one row past it (reallocated).  score_assign and a staged pass of B against a fresh
    context and the oracle."""
    w = world("plain")
    a, fits, grows = rc.growth_steps(w)
    fx_b = rc.Fixture("steps", fits if b == "fits" else grows)
    stride = rc.slab_stride(w.topo.n)
    cap = rc.grow(8 * stride)
    assert (int(fx_b.blob[5]) * stride <= cap) == (b == "fits")
    for kind in ("steps", "score_assign"):
        exp = expected("plain", kind, "growth_" + b, fx=fx_b)
        eng = make_engine(w)
        try:
            run(kind, eng, w, rc.Fixture("steps", a))
            same(run(kind, eng, w, fx_b), exp, (b, kind))
        finally:
            eng.close()


# ---- 2. failed calls in between

FAILING = [(x, "plain") for x in rc.FAILING_NAMES] + [(x, "level0") for x in rc.ELIMIT_NAMES]


@pytest.mark.parametrize("name,wname", FAILING, ids=[f[0] for f in FAILING])
def test_failed_call_then_every_kind(name, wname):
    """A call that fails after its blob was uploaded to the batch (EINVAL at the blob's last word, ELIMIT on a
    context without the level flags, EINEXACT at the exactness bound of the ranking and of the pod waves), then every
    kind with both fixtures, each behind another failure."""
    w = world(wname)
    cases = {x[0]: x[1:] for x in (rc.failing(w) if wname == "plain" else rc.failing_levels(w))}
    entry, args, code = cases[name]
    eng = make_engine(w)
    try:
        for kind in rc.KINDS:
            for size in rc.SIZES:
                with pytest.raises(RbgTopoError) as e:
                    getattr(eng, entry)(*args)
                assert e.value.code == code, (name, e.value)
                run_checked(eng, wname, kind, size, (name, kind, size))
    finally:
        eng.close()


# ---- 3. topology changes under the pool

def test_topology_changes_every_kind():
    """set_topology with N = 4 097 -> 129 -> 65 537 -> 4 097: the pool's batches were sized against the old slab
    stride; every kind with both fixtures after each change."""
    first = world(f"topo{rc.TOPO_SEQUENCE[0]}")
    eng = make_engine(first)
    try:
        for i, n in enumerate(rc.TOPO_SEQUENCE):
            wname = f"topo{n}"
            t = world(wname).topo
            if i:
                eng.set_topology(t.row_ptr, t.col_idx, t.edge_w, t.free, t.domain, t.domain_owner)
            for kind in rc.KINDS:
                for size in ("large", "small"):
                    run_checked(eng, wname, kind, size, (i, n, kind, size))
    finally:
        eng.close()


# ---- a world = 2 pair of contexts on one device

WORLD2_KINDS = ("score_assign", "steps", "direct", "staged", "committed")   # the kinds that accept world > 1
REFUSED_WORLD2 = ("ranked", "committed_ranked", "lw", "lw_ranked", "lw_committed", "lw_committed_ranked")


def test_world2_pair_of_contexts():
    """Rank 0 and rank 1 of one world = 2 snapshot, two contexts on one device: half slabs of the dense matrix,
    replicated selection, and place_groups on the staged path with its pre-validation upload and early emit.  On each
    rank every ordered pair of the kinds that accept world > 1 (large then small, small then large), each pair behind
    a ranked or leader-worker call the context refuses with ELIMIT; every call against a fresh world = 2 context of
    the same rank, and its placements against the world = 1 results."""
    wname = "plain"
    w = world(wname)
    engs = [make_engine(w, rank=r, n_ranks=2) for r in range(2)]
    placements = ("assign", "status", "domain", "rounds")
    k = 0
    try:
        for a in WORLD2_KINDS:
            for b in WORLD2_KINDS:
                for sa, sb in (("large", "small"), ("small", "large")):
                    for r, eng in enumerate(engs):
                        refused = REFUSED_WORLD2[k % len(REFUSED_WORLD2)]
                        k += 1
                        with pytest.raises(RbgTopoError) as e:
                            run(refused, eng, w, w.fixture(refused, sa))
                        assert e.value.code == -6, (refused, e.value)
                        for kind, size in ((a, sa), (b, sb)):
                            tag = (r, a, sa, b, sb, kind)
                            got = run(kind, eng, w, w.fixture(kind, size))
                            same(got, expected(wname, kind, size, rank=r, n_ranks=2), tag)
                            one = expected(wname, kind, size)
                            same({n: got[n] for n in placements if n in got},
                                 {n: one[n] for n in placements if n in one}, tag + ("world 1",))
    finally:
        for eng in engs:
            eng.close()


# ---- 4. a seeded sequence on the level context

def _refreshes(w, rng, count):
    """update_nodes, update_nodes_delta and an occupancy refresh (partitions kept), in turn."""
    import levels_oracle as lo
    n = w.topo.n
    out, free = [], w.topo.free.copy()
    gids = sorted({g.gid for g in w.fx[("groups", "large")].groups})
    for k in range(count):
        gen = 10 + k
        if k % 3 == 0:
            free = np.where(rng.random(n) < 0.2, 0, w.topo.free).astype(np.int32)
            out.append(lambda e, f=free, g=gen: e.update_nodes(f, None, generation=g))
        elif k % 3 == 1:
            nodes = np.sort(rng.choice(n, size=24, replace=False)).astype(np.int32)
            vals = ((free[nodes] + 1) % 4).astype(np.int32)
            free = free.copy()
            free[nodes] = vals
            out.append(lambda e, nd=nodes, v=vals, g=gen: e.update_nodes_delta(nd, v, generation=g))
        else:
            occ = lo.random_occ(rng, n, 3, gids[:4] + [999], max(1, n // 6))
            out.append(lambda e, o=occ, g=gen: e.set_exclusive_levels(None, o, generation=g))
    return out


def test_seeded_sequence_with_refreshes_and_held_handles():
    """400 calls drawn from K x fixtures on the level context, with a refresh every ~70 calls, two staged handles
    (steps, groups) held across the sequence and re-run at random points, and kernel timing switched on halfway; every
    call against a fresh context with the same refresh history, every re-run of a held handle against its pass there.
    A timed run_staged(h, 3) + fetch reports three passes' kernel times."""
    wname = "levels"
    w = world(wname)
    rng = np.random.default_rng(2026)
    refresh = _refreshes(w, rng, 5)
    at = {70 * (k + 1): k for k in range(len(refresh))}
    eng = make_engine(w)
    held = {"steps": (eng.stage(w.fx[("steps", "large")].blob), w.fx[("steps", "large")]),
            "staged": (eng.stage_groups(w.fx[("groups", "small")].blob), w.fx[("groups", "small")])}
    version, timing, reruns = 0, False, 0
    try:
        for i in range(400):
            if i in at:
                refresh[at[i]](eng)
                version += 1
            if i == 200:
                eng.set_kernel_timing(True)
                timing = True
                h, fx = held["staged"]
                eng.run_staged(h, 3)
                eng.fetch(h)
                sc, se = eng.last_pass_times()
                assert len(sc) == len(se) == 3, (sc, se)
                assert (sc > 0).all() and (se > 0).all() and np.isfinite(sc).all() and np.isfinite(se).all(), (sc, se)
            kw = dict(version=version, refreshes=tuple(refresh[:version]), timing=timing)
            if rng.random() < 0.1:
                which = ("steps", "staged")[int(rng.integers(0, 2))]
                h, fx = held[which]
                eng.run_staged(h, 1)
                got = staged_result(eng, w, fx, h)
                size = "large" if which == "steps" else "small"
                same(got, expected(wname, which, size, **kw), (i, "held", which, version, timing))
                reruns += 1
            kind = rc.KINDS[int(rng.integers(0, len(rc.KINDS)))]
            size = rc.SIZES[int(rng.integers(0, 2))]
            run_checked(eng, wname, kind, size, (i, kind, size, version, timing), **kw)
        assert reruns >= 20, reruns
        for h, _ in held.values():
            eng.release(h)
    finally:
        eng.close()


# ---- 5. threads

@pytest.mark.parametrize("n_threads", [4, 8])
def test_threads_share_one_context(n_threads):
    """Threads (ctypes releases the GIL) on one context, each with its own seeded sequence of kinds and fixtures and
    no refresh: the pool hands its batches between entry points in any order.  Outputs against the fresh context
    (the counters are the context's last call, whichever thread made it)."""
    wname = "plain"
    w = world(wname)
    for kind in rc.KINDS:
        for size in rc.SIZES:
            expected(wname, kind, size)
    eng = make_engine(w)
    errors, done = [], []

    def worker(t):
        rng = np.random.default_rng(500 + t)
        try:
            for i in range(40):
                kind = rc.KINDS[int(rng.integers(0, len(rc.KINDS)))]
                size = rc.SIZES[int(rng.integers(0, 2))]
                same(run(kind, eng, w, w.fixture(kind, size), counters=False), expected(wname, kind, size),
                     (t, i, kind, size))
            done.append(t)
        except BaseException as e:   # reported below, in the test's thread
            errors.append((t, repr(e)[:2000]))

    try:
        ths = [threading.Thread(target=worker, args=(t,)) for t in range(n_threads)]
        for th in ths:
            th.start()
        for th in ths:
            th.join()
        assert not errors, errors[:2]
        assert sorted(done) == list(range(n_threads))
    finally:
        eng.close()
