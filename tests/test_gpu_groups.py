"""GPU: whole-group placement (rbgtopo_place_groups, the C++ level/wave loop behind
the ABI) against the same loop run in Python over the CPU oracle, and the plugin
mirror end to end."""
import numpy as np
import pytest

from rbg_b200 import synth
from rbg_b200.plugin import (EXCLUSIVE_TOPOLOGY_KEY, GANG_SCHEDULING_KEY, B200TopoPodGroupManager, RoleBasedGroup,
                             RoleSpec)

pytestmark = pytest.mark.gpu


def _fleet(n_nodes, n_groups, seed, excl_every=0, gang_every=0, big_every=0):
    shapes = [synth.shape_mooncake(), synth.shape_pd_144(), synth.shape_fleet8(), synth.shape_sglang_pd()]
    out = []
    for g in range(n_groups):
        sh = shapes[g % len(shapes)]
        roles = [RoleSpec(r.name, r.replicas, tuple(r.deps), r.demand) for r in sh.roles]
        if big_every and g % big_every == 0:
            roles[1].replicas = 41                     # forces waves of 32 + 9
        ann = {}
        if excl_every and g % excl_every == 0:
            ann[EXCLUSIVE_TOPOLOGY_KEY] = "topology.kubernetes.io/nvlink-domain"
        if gang_every and g % gang_every == 0:
            ann[GANG_SCHEDULING_KEY] = "true"
        placed = [(sh.roles[q].name, node) for node, q, _ in synth.random_anchors(n_nodes, len(sh.roles), g % 3, seed, g)]
        out.append(RoleBasedGroup("default", f"rbg{g}", roles, annotations=ann, gid=g, policy_rules=sh.policy_rules,
                                  placed=placed))
    return out


def _oracle_manager(topo):
    from test_plugin_host import OraclePlacer
    return B200TopoPodGroupManager(OraclePlacer(topo))


@pytest.mark.parametrize("n,kw", [(1024, {}), (4096, dict(excl_every=3, gang_every=4)), (2048, dict(big_every=5)),
                                  (10000, dict(excl_every=5))])
def test_place_groups_matches_oracle_wave_loop(n, kw):
    from gpu_util import new_engine
    topo = synth.make_topology(n, seed=n + 1, tiers=4, owned_frac=0.2 if kw.get("excl_every") else 0.0)
    rbgs = _fleet(n, 40, seed=7, **kw)
    eng = new_engine(topo)
    got = B200TopoPodGroupManager(eng).reconcile_pod_groups(rbgs)               # C++ loop, CUDA kernels
    got_py = B200TopoPodGroupManager(eng).reconcile_pod_groups_by_waves(rbgs)   # Python loop, CUDA kernels
    ref = _oracle_manager(topo).reconcile_pod_groups_by_waves(rbgs)             # Python loop, CPU oracle
    for a, b, c in zip(got, got_py, ref):
        assert a.nodes == c.nodes and b.nodes == c.nodes
        assert a.status == c.status == b.status
        assert a.domain == c.domain == b.domain
    eng.close()


def test_scarce_cluster_gang_groups_fail_atomically():
    from gpu_util import new_engine
    topo = synth.make_topology(512, seed=2, tiers=2, max_free=1)
    topo.free[5:] = 0                      # at most 5 slots in the whole cluster
    rbgs = _fleet(512, 12, seed=3, gang_every=2)
    eng = new_engine(topo)
    got = B200TopoPodGroupManager(eng).reconcile_pod_groups(rbgs)
    ref = _oracle_manager(topo).reconcile_pod_groups_by_waves(rbgs)
    assert any(p.status == 2 for p in ref)
    for a, c in zip(got, ref):
        assert a.nodes == c.nodes and a.status == c.status
    eng.close()


def test_concurrent_callers_share_one_context():
    """Up to --max-concurrent-reconciles goroutines call the plugin at once
    (cmd/rbgs/main.go:140-143): 10 threads on one ctx, identical results."""
    import threading
    from gpu_util import new_engine
    topo = synth.make_topology(4096, seed=6, tiers=4)
    eng = new_engine(topo)
    mgr = B200TopoPodGroupManager(eng)
    fleets = [_fleet(4096, 6, seed=100 + t) for t in range(10)]
    blobs = [mgr.groups_blob(f)[0] for f in fleets]
    want = [eng.place_groups(b) for b in blobs]
    got = [None] * 10
    errs = []

    def work(i):
        try:
            for _ in range(5):
                got[i] = eng.place_groups(blobs[i])
        except Exception as e:   # pragma: no cover
            errs.append(e)
    th = [threading.Thread(target=work, args=(i,)) for i in range(10)]
    [t.start() for t in th]
    [t.join() for t in th]
    assert not errs
    for g, w in zip(got, want):
        assert all(np.array_equal(x, y) for x, y in zip(g, w))
    eng.close()


def test_degenerate_fleets():
    """No groups, groups with nothing pending, a single one-replica group: the plan machinery
    (device expansion, zero-sized launches) must cope."""
    from gpu_util import new_engine
    topo = synth.make_topology(700, seed=4, tiers=3)
    eng = new_engine(topo)
    mgr = B200TopoPodGroupManager(eng)
    assert mgr.reconcile_pod_groups([]) == []
    idle = RoleBasedGroup("default", "idle", [RoleSpec("a", 0, (), 1), RoleSpec("b", 0, ("a",), 1)], gid=0)
    one = RoleBasedGroup("default", "one", [RoleSpec("a", 1, (), 1)], gid=1)
    for fleet in ([idle], [idle, one, idle], [one]):
        got = mgr.reconcile_pod_groups(fleet)
        ref = _oracle_manager(topo).reconcile_pod_groups_by_waves(fleet)
        for a, c in zip(got, ref):
            assert a.nodes == c.nodes and a.status == c.status and a.domain == c.domain
    eng.close()


def test_churn_reconcile_matches_oracle():
    """BASELINE.json configs[4]: continuous reconcile under churn — every step 10 % of the nodes
    leave (capacity 0) or come back, the snapshot is refreshed asynchronously
    (rbgtopo_update_nodes) and the whole fleet is re-placed; each step equals the oracle run
    on that step's snapshot."""
    from gpu_util import new_engine
    n = 4000
    topo = synth.make_topology(n, seed=21, tiers=4)
    free0 = topo.free.copy()
    rbgs = _fleet(n, 32, seed=8, gang_every=5)
    eng = new_engine(topo)
    mgr = B200TopoPodGroupManager(eng)
    rng = np.random.default_rng(5)
    gone = np.zeros(n, dtype=bool)
    for step in range(4):
        flip = rng.choice(n, size=n // 10, replace=False)
        gone[flip] = ~gone[flip]
        topo.free = np.where(gone, 0, free0).astype(np.int32)
        eng.update_nodes(topo.free, None, generation=10 + step)
        got = mgr.reconcile_pod_groups(rbgs)
        ref = _oracle_manager(topo).reconcile_pod_groups_by_waves(rbgs)
        for a, c in zip(got, ref):
            assert a.nodes == c.nodes and a.status == c.status and a.domain == c.domain, step
        assert not any(gone[v] for p in got for v in p.nodes.values() if v >= 0)   # nobody lands on a removed node
    eng.close()


def test_plan_dense_matrix_and_lists_match_oracle_per_wave():
    """A staged multi-wave plan leaves the same dense matrix rows and top-K lists in HBM as
    the wave-by-wave oracle run (rows: wave-major, groups in order)."""
    from gpu_util import new_engine
    from oracle import placer as oracle_placer
    from rbg_b200.blob import BlobBuilder
    from rbg_b200.plugin import _GroupRun
    n = 3000
    topo = synth.make_topology(n, seed=11, tiers=4, owned_frac=0.2)
    rbgs = _fleet(n, 24, seed=5, excl_every=3, big_every=5)
    eng = new_engine(topo)
    mgr = B200TopoPodGroupManager(eng)
    gblob, _ = mgr.groups_blob(rbgs)
    h = eng.stage_groups(gblob)
    eng.run_staged(h, 1)
    eng.fetch(h)
    runs = [_GroupRun(r, mgr.arith) for r in rbgs]
    from gpu_util import plan_rows
    row_of = plan_rows(gblob, topo)          # dense rows: group order; top-K lists (role rows): wave-major
    index_of = {id(g): i for i, g in enumerate(runs)}
    rr = w = 0
    while True:
        active = [g for g in runs if w < len(g.waves)]
        if not active:
            break
        bb = BlobBuilder()
        for g in active:
            bb.add(g.step(w))
        ref = oracle_placer.place(topo, bb.build(), want_matrix=True, want_topk=True)
        assert ref["rc"] == 0 and (ref["status"] == 0).all()     # nobody fails: rows stay aligned with the plan
        off = 0
        for g in active:
            cnt = sum(c for _, _, c in g.waves[w].roles)
            row0 = row_of[(index_of[id(g)], w)]
            for k in range(cnt):
                got = eng.read_scores(h, row0 + k)
                exp = ref["matrix"][off + k]
                bad = np.nonzero(got.view(np.uint32) != exp.view(np.uint32))[0]
                assert len(bad) == 0, (w, off + k, len(bad), int(bad[0]), float(got[bad[0]]), float(exp[bad[0]]))
            off += cnt
        for i in range(ref["topk"].shape[0]):
            assert np.array_equal(eng.read_topk(h, rr + i, 32), ref["topk"][i]), (w, i)
        off = 0
        for i, g in enumerate(active):
            cnt = sum(c for _, _, c in g.waves[w].roles)
            g.absorb(w, ref["assign"][off:off + cnt], int(ref["status"][i]), int(ref["domain"][i]), n)
            off += cnt
        rr += ref["topk"].shape[0]
        w += 1
    assert w >= 3
    eng.release(h)
    eng.close()


def test_chained_batches_equal_separate_runs():
    """rbgtopo_run_staged_chain: passes round robin over distinct staged batches, the dense-matrix kernel of a pass
    chained behind the selection kernel of the pass before it (programmatic dependent launch).  Every batch must end
    with exactly what a plain rbgtopo_run_staged leaves: placements, status, domains and every dense-matrix row —
    also for tiny batches (few dense-matrix CTAs: the ordering argument must not lean on the grid size), for a single
    handle, and with kernel timing on (the documented fallbacks)."""
    from gpu_util import new_engine
    n = 3000
    topo = synth.make_topology(n, seed=11, tiers=4, owned_frac=0.2)
    eng = new_engine(topo)
    mgr = B200TopoPodGroupManager(eng)
    fleets = [_fleet(n, 24, seed=5, excl_every=3, big_every=5), _fleet(n, 40, seed=9, excl_every=4, big_every=7),
              _fleet(n, 2, seed=3, excl_every=2, big_every=0), _fleet(n, 1, seed=4, excl_every=0, big_every=0)]
    blobs = [mgr.groups_blob(f)[0] for f in fleets]
    want = []
    for gb in blobs:                      # reference: each batch alone
        h = eng.stage_groups(gb)
        eng.run_staged(h, 1)
        a, st, dm = eng.fetch(h)
        rows = [eng.read_scores(h, r).copy() for r in range(int(gb[4]))]
        want.append((a.copy(), st.copy(), dm.copy(), rows))
        eng.release(h)

    def check(hs, which):
        for h, i in zip(hs, which):
            a, st, dm = eng.fetch(h)
            wa, ws, wd, wrows = want[i]
            assert np.array_equal(a, wa) and np.array_equal(st, ws) and np.array_equal(dm, wd), i
            for r, exp in enumerate(wrows):
                got = eng.read_scores(h, r)
                assert np.array_equal(got.view(np.uint32), exp.view(np.uint32)), (i, r)

    hs = [eng.stage_groups(gb) for gb in blobs]
    eng.run_staged_chain(hs, 4)           # one pass each
    check(hs, range(4))
    eng.run_staged_chain(hs, 4 * 7 + 2)   # many rounds, ending mid-round
    check(hs, range(4))
    eng.run_staged_chain(hs[2:], 9)       # the two tiny batches alone (1-2 groups: a handful of CTAs per kernel)
    check(hs[2:], [2, 3])
    eng.run_staged_chain(hs[:1], 3)       # one handle: plain passes
    check(hs[:1], [0])
    eng.set_kernel_timing(True)           # per-kernel events: plain passes
    eng.run_staged_chain(hs, 8)
    check(hs, range(4))
    eng.set_kernel_timing(False)
    with pytest.raises(Exception):
        eng.run_staged_chain([hs[0], hs[0]], 2)
    for h in hs:
        eng.release(h)
    eng.close()


def test_place_groups_rejects_bad_blobs_and_recovers():
    """Malformed GROUPS blobs through rbgtopo_place_groups: the same error codes on the direct path (default) and on the
    staged one (the subprocess variant RBGTOPO_NO_DIRECT runs this test too), nothing placed, and the context keeps
    working — the direct path has enqueued the upload (and, for errors of the second validation pass, the dense matrix)
    by the time it finds them."""
    from gpu_util import new_engine
    from rbg_b200.engine import RbgTopoError
    n = 2048
    topo = synth.make_topology(n, seed=6, tiers=3)
    eng = new_engine(topo)
    mgr = B200TopoPodGroupManager(eng)
    gb, _ = mgr.groups_blob(_fleet(n, 12, seed=2, excl_every=4, gang_every=5))
    gb = np.ascontiguousarray(gb, dtype=np.int32)
    good = eng.place_groups(gb)
    HDR, GW = 8, 12

    def rec(g):
        return HDR + g * GW

    def mutate(f):
        b = gb.copy()
        f(b)
        return b

    def set_(idx, v):
        return lambda b: b.__setitem__(idx, v)

    g3 = rec(3)
    roles3, pair3, anc_n3, anc3 = int(gb[g3 + 4]), int(gb[g3 + 5]), int(gb[g3 + 6]), int(gb[g3 + 7])
    cases = [
        (set_(0, 0x12345), -1),                                   # magic
        (set_(g3 + 3, 0), -6),                                    # q = 0 roles: limit
        (set_(g3 + 3, 17), -6),                                   # q > 16
        (set_(roles3 + 1, -2), -1),                               # pending < 0
        (set_(roles3 + 2, 1 << 20), -1),                          # demand out of range
        (set_(roles3 + 3, 0x40), -1),                             # unknown role flag
        (set_(pair3, -1), -1),                                    # pair weight < 0
        (set_(g3 + 1, 0x100), -1),                                # unknown group flags
        (set_(g3 + 8, int(gb[g3 + 8]) + 1), -1),                  # assign_off does not continue the prefix
        (set_(g3 + 2, 1 << 20), -1),                              # fixed_domain out of range
    ]
    g_anc = next(g for g in range(12) if int(gb[rec(g) + 6]) > 0)
    a_off = int(gb[rec(g_anc) + 7])
    q_anc, pair_anc, role_anc = int(gb[rec(g_anc) + 3]), int(gb[rec(g_anc) + 5]), int(gb[a_off + 1])
    cases += [
        (set_(pair_anc + 0 * q_anc + role_anc, 1 << 23), -4),     # exactness bound: anchor weight x row weight >= 2^24
        (set_(a_off, n + 5), -1),                                 # scheduled pod on a node that does not exist
        (set_(a_off + 1, 99), -1),                                # ... of a role that does not exist
        (set_(a_off + 2, (1 << 24) + 1), -1),                     # ... with an inadmissible count
    ]
    for f, code in cases:
        bad = mutate(f)
        with pytest.raises(RbgTopoError) as ei:
            eng.place_groups(bad)
        assert ei.value.code == code, (code, str(ei.value))
        again = eng.place_groups(gb)                              # the context is unharmed
        assert all(np.array_equal(x, y) for x, y in zip(again, good))
    eng.close()


@pytest.mark.parametrize("var", ["RBGTOPO_VERIFY_PLAN", "RBGTOPO_PER_WAVE_PLAN", "RBGTOPO_SPLIT_MIN_GROUPS",
                                 "RBGTOPO_CONCURRENT_PLAN", "RBGTOPO_EMIT_TMA", "RBGTOPO_CONCURRENT_PLAN+RBGTOPO_EMIT_TMA",
                                 "RBGTOPO_EMIT_STEPS+RBGTOPO_VERIFY_PLAN", "RBGTOPO_KERNEL_TIMING", "RBGTOPO_NO_PDL",
                                 "RBGTOPO_EMIT_ROWS", "RBGTOPO_NO_DIRECT"])
def test_plan_variants_in_a_subprocess(var):
    """The library reads its switches when it loads, hence the subprocess.
    RBGTOPO_VERIFY_PLAN: every place_groups / stage_groups call compares the plan k_expand_plan
    wrote in HBM (and the host-side geometry) word for word with the host plan builder.
    RBGTOPO_PER_WAVE_PLAN: the fallback that runs one launch per wave and chains placements
    through the plan blob (what groups too large for k_plan_group's shared memory take).
    RBGTOPO_SPLIT_MIN_GROUPS=1 (-> 2): place_groups pipelines every fleet as two halves (opt-in).
    RBGTOPO_CONCURRENT_PLAN: k_plan_group in record mode on a second stream + k_plan_correct (opt-in).
    RBGTOPO_EMIT_TMA: the dense rows of plans through k_emit_tma (TMA bulk stores) instead of k_emit_rows.
    RBGTOPO_EMIT_STEPS: the step-major dense-matrix kernel (k_score_emit<false, ETAB>) instead of k_emit_rows.
    RBGTOPO_KERNEL_TIMING / RBGTOPO_NO_PDL: an event between the two plan kernels / plain stream order instead of the
    programmatic dependent launch.  RBGTOPO_EMIT_ROWS=1: one row per segment of k_emit_rows (the smallest segment).
    RBGTOPO_NO_DIRECT: rbgtopo_place_groups through the staged path (expanded plan, early emit) that world > 1 takes.
    Each variant runs this file and tests/test_gpu_groups_limits.py (8-role waves, 16-role groups, ragged node counts)."""
    import os
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ)
    for v in var.split("+"):
        env[v] = "1"
    r = subprocess.run(
        [sys.executable, "-m", "pytest", "tests/test_gpu_groups.py", "tests/test_gpu_groups_limits.py", "-q", "-m", "gpu", "-x",
         "-k", "not subprocess"],
        cwd=root, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert "passed" in r.stdout


def test_bench_shape_plan_parity():
    """The plan bench.py times (cfg3: 1 024 mooncake RBGs x 10 000 nodes, all 3 waves) against the
    CPU oracle's wave loop: dense matrix bits of every replica row of 128 sampled groups, and the
    assignment / status / domain of those groups — the checker bench.py itself runs before timing."""
    import bench
    from gpu_util import new_engine
    n, groups = 10000, 1024
    topo = synth.make_topology(n, seed=0, tiers=4, samples_per_tier=5)
    specs = bench.fleet_spec("mooncake", groups, n)
    eng = new_engine(topo)
    gblob, _ = B200TopoPodGroupManager(eng).groups_blob(bench.to_plugin(specs))
    h = eng.stage_groups(gblob)
    eng.run_staged(h, 1)
    fetched = eng.fetch(h)
    sample = sorted(set(int(i) for i in np.linspace(0, groups - 1, 128)))
    par = bench.parity_check(eng, topo, specs, gblob, h, fetched, sample, 0, n, 8)
    assert par["ok"] and par["rows_checked"] == 128 * 7 and par["waves"] == 3, par
    # the whole fleet's placements through the host-buffer entry point equal the staged plan's
    a, s, d = eng.place_groups(gblob)
    assert np.array_equal(a, fetched[0]) and np.array_equal(s, fetched[1]) and np.array_equal(d, fetched[2])
    eng.release(h)
    eng.close()


def test_exclusive_group_with_nothing_pending_confirms_its_domain():
    """ADVICE r1: plan path and host loop agree on the result contract — an exclusive group that
    already occupies a domain and has no pending replica reports that domain."""
    from gpu_util import new_engine
    topo = synth.make_topology(512, seed=3, tiers=2)
    eng = new_engine(topo)
    mgr = B200TopoPodGroupManager(eng)
    ann = {EXCLUSIVE_TOPOLOGY_KEY: "topology.kubernetes.io/nvlink-domain"}
    idle = RoleBasedGroup("default", "idle", [RoleSpec("a", 2, (), 1)], annotations=ann, gid=5, current={"a": 2},
                          placed=[("a", 16), ("a", 17)], exclusive_domain=2)
    busy = RoleBasedGroup("default", "busy", [RoleSpec("a", 3, (), 1)], annotations=ann, gid=6, current={"a": 1},
                          placed=[("a", 40)], exclusive_domain=5)
    got = mgr.reconcile_pod_groups([idle, busy])
    ref = _oracle_manager(topo).reconcile_pod_groups_by_waves([idle, busy])
    assert got[0].domain == 2 and got[0].nodes == {} and got[0].status == 0
    assert got[1].domain == ref[1].domain == 5 and got[1].nodes == ref[1].nodes
    eng.close()
