"""GPU: committed batches (rbgtopo_place_groups_committed, DESIGN.md §3.8) bit-equal to the oracle's committed loop
(tests/committed_oracle.py) run on the very same GROUPS blob — assign, status and domain of every group — on contended
batches, exclusive races, scarce capacity, partially placed groups, the ABI limits of tests/groups_gen.py and the bench
fleet; plus the call's contract: rounds, one-group batches, world = 2, concurrent callers, malformed blobs, the
RBGTOPO_ELIMIT path, and snapshot-semantics calls on the same context left as they were."""
import threading

import numpy as np
import pytest

import groups_gen as gg
from committed_oracle import result_arrays, run_fleet_committed
from oracle import wave_loop
from rbg_b200 import synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, STEP_GANG, Group, GroupsBuilder
from rbg_b200.engine import RbgTopoError, TopoPlacer

pytestmark = pytest.mark.gpu


def engine(topo, **kw):
    eng = TopoPlacer(device=0, **kw)
    eng.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    return eng


def pending_groups(gblob):
    return sum(1 for g in range(int(gblob[2])) if int(gblob[8 + 12 * g + 9]) > 0)


def check(eng, topo, gblob, fast=False):
    """The committed call against the oracle; returns (assign, status, domain, rounds)."""
    a, s, d, rounds = eng.place_groups_committed(gblob)
    groups = wave_loop.groups_from_blob(gblob)
    states = run_fleet_committed(topo, groups, fast=fast)
    ea, es, ed = result_arrays(states)
    n = len(states)
    assert np.array_equal(a[:len(ea)], ea), np.nonzero(a[:len(ea)] != ea)[0][:8]
    assert np.array_equal(s[:n], es), (s[:n], es)
    assert np.array_equal(d[:n], ed), (d[:n], ed)
    ng = int(gblob[2])
    assert (rounds == 0) if pending_groups(gblob) == 0 else (1 <= rounds <= ng), (rounds, ng)
    return a, s, d, rounds


def _build(groups):
    gb = GroupsBuilder()
    for g in groups:
        gb.add(g)
    return gb.build()


def contended_case(seed, exclusive_all=False):
    """Few nodes, many similar groups: levels, gang and non-gang under scarce capacity, exclusive groups racing for the
    same domains, preset and self-owned domains, fixed domains, shared gids, scheduled pods."""
    rng = np.random.default_rng(seed)
    n = int(rng.integers(6, 48))
    topo = synth.make_topology(n, seed=seed + 11, tiers=2, owned_frac=0.2 if n >= 16 else 0.0, max_free=3)
    if rng.random() < 0.5:
        topo.free = np.where(rng.random(n) < 0.5, 0, topo.free).astype(np.int32)
    n_dom = len(topo.domain_owner)
    row_w = gg.wsum_max(topo)
    ng = int(rng.integers(4, 20))
    groups = []
    for g in range(ng):
        q = int(rng.integers(1, 4))
        lv = np.sort(rng.integers(0, 2, size=q))
        roles = [(int(lv[i]), int(rng.integers(0, 6)), int(rng.choice([0, 1, 1, 2])),
                  ROLE_EXCLUSIVE if rng.random() < 0.8 else 0) for i in range(q)]
        pair = rng.integers(0, 3, size=(q, q))
        np.fill_diagonal(pair, 1)
        excl = exclusive_all or rng.random() < 0.4
        gid = 100 + (int(rng.integers(0, g)) if g and rng.random() < 0.15 else g)
        fixed = int(rng.integers(0, n_dom)) if excl and rng.random() < 0.2 else -1
        if excl and rng.random() < 0.2:
            topo.domain_owner[int(rng.integers(0, n_dom))] = gid
        anchors = [(int(rng.integers(0, n)), int(rng.integers(0, q)), 1) for _ in range(int(rng.integers(0, 3)))]
        grp = Group(gid=gid, roles=roles, pair=pair.tolist(), anchors=anchors,
                    flags=(STEP_EXCLUSIVE if excl else 0) | (STEP_GANG if rng.random() < 0.4 else 0), fixed_domain=fixed)
        while not gg.exact_ok(grp, row_w):
            p = np.asarray(grp.pair)
            p[np.unravel_index(int(np.argmax(p)), p.shape)] -= 1
            grp.pair = p.tolist()
        groups.append(grp)
    return topo, _build(groups)


def test_contended_batches_match_oracle():
    """100 seeds of small contended batches."""
    stats = {"rounds": [], "status1": 0, "status2": 0, "excl": 0}
    for seed in range(100):
        topo, gblob = contended_case(seed, exclusive_all=seed % 4 == 0)
        eng = engine(topo)
        try:
            _, s, d, rounds = check(eng, topo, gblob)
        finally:
            eng.close()
        stats["rounds"].append(rounds)
        stats["status1"] += int((s == 1).sum())
        stats["status2"] += int((s == 2).sum())
        stats["excl"] += int((d >= 0).sum())
    # the seeds reach partial groups, failed gangs, exclusive domains and more than one round
    assert stats["status1"] and stats["status2"] and stats["excl"] and max(stats["rounds"]) > 1, stats


@pytest.mark.parametrize("seed,n,scarce,excl", gg.CASES)
def test_generated_fleets_at_the_abi_limits(seed, n, scarce, excl):
    case = gg.make_case(seed, n, scarce=scarce, exclusive=excl)
    eng = engine(case.topo)
    try:
        check(eng, case.topo, case.blob)
    finally:
        eng.close()


def test_bench_fleet_mooncake_1024_groups_10000_nodes():
    """cfg3's fleet as one committed batch: all 1 024 groups against the oracle (its fast variant, about 1 s on one CPU
    thread), no node over-committed."""
    import bench
    from rbg_b200.plugin import B200TopoPodGroupManager
    topo = synth.make_topology(10000, seed=0)
    specs = bench.fleet_spec("mooncake", 1024, 10000, 0)
    eng = engine(topo)
    try:
        gblob, _ = B200TopoPodGroupManager(eng).groups_blob(bench.to_plugin(specs))
        a, s, d, rounds = check(eng, topo, gblob, fast=True)
        groups = wave_loop.groups_from_blob(gblob)
        used = np.zeros(topo.n, dtype=np.int64)
        off = 0
        for g in groups:
            for r in g.roles:
                sl = a[off:off + r.replicas]
                np.add.at(used, sl[sl >= 0], r.demand)
                off += r.replicas
        assert (used <= topo.free).all()
        assert rounds >= 2
    finally:
        eng.close()


def test_rounds_and_one_group_batches():
    """A batch whose groups never read what another took needs one round; a one-group batch equals place_groups."""
    topo = synth.make_topology(512, seed=5, tiers=2, max_free=4)
    topo.domain_owner[:] = -1
    doms = np.random.default_rng(5).permutation(len(topo.domain_owner))[:12]
    groups = [Group(gid=40 + i, roles=[(0, 2, 1, ROLE_EXCLUSIVE), (1, 3, 1, ROLE_EXCLUSIVE)], pair=[[1, 1], [1, 1]],
                    anchors=[], flags=STEP_EXCLUSIVE, fixed_domain=int(dm)) for i, dm in enumerate(doms)]
    eng = engine(topo)
    try:
        gblob = _build(groups)
        a, s, d, rounds = check(eng, topo, gblob)
        assert rounds == 1 and list(d) == [int(x) for x in doms]
        assert np.array_equal(a, eng.place_groups(gblob)[0])
        topo2, gblob2 = contended_case(3)
        eng.set_topology(topo2.row_ptr, topo2.col_idx, topo2.edge_w, topo2.free, topo2.domain, topo2.domain_owner)
        for grp in _groups_of(gblob2)[:6]:
            one = _build([grp])
            a1, s1, d1, r1 = eng.place_groups_committed(one)
            a2, s2, d2 = eng.place_groups(one)
            assert np.array_equal(a1, a2) and np.array_equal(s1, s2) and np.array_equal(d1, d2)
            assert r1 == (1 if pending_groups(one) else 0)
    finally:
        eng.close()


def _groups_of(gblob):
    """The Group records of a GROUPS blob (to rebuild sub-batches)."""
    b = np.asarray(gblob, dtype=np.int64)
    out = []
    for i in range(int(b[2])):
        gid, flags, fixed, q, role_off, pair_off, na, anchor_off = (int(x) for x in b[8 + 12 * i:][:8])
        roles = [tuple(int(x) for x in b[role_off + 4 * r:role_off + 4 * r + 4]) for r in range(q)]
        pair = b[pair_off:pair_off + q * q].reshape(q, q).tolist()
        anchors = [tuple(int(x) for x in b[anchor_off + 3 * a:anchor_off + 3 * a + 3]) for a in range(na)]
        out.append(Group(gid=gid, roles=roles, pair=pair, anchors=anchors, flags=flags, fixed_domain=fixed))
    return out


def test_world_2_contexts_and_concurrent_callers():
    topo, gblob = contended_case(7)
    ref = None
    eng = engine(topo)
    try:
        ref = check(eng, topo, gblob)
        results = [None] * 10

        def call(i):
            results[i] = eng.place_groups_committed(gblob)
        threads = [threading.Thread(target=call, args=(i,)) for i in range(10)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        for r in results:
            assert all(np.array_equal(x, y) for x, y in zip(r[:3], ref[:3])) and r[3] == ref[3]
    finally:
        eng.close()
    engs = [engine(topo, rank=r, world=2) for r in range(2)]
    try:
        for e in engs:
            r = e.place_groups_committed(gblob)
            assert all(np.array_equal(x, y) for x, y in zip(r[:3], ref[:3])) and r[3] == ref[3]
    finally:
        for e in engs:
            e.close()


def _code(fn):
    try:
        fn()
    except RbgTopoError as e:
        return e.code
    return 0


def test_malformed_blobs_same_codes_as_place_groups_and_recovery():
    topo, gblob = contended_case(11)
    eng = engine(topo)
    try:
        good = check(eng, topo, gblob)
        rec = 8   # group 0's record
        role_off, anchor_off = int(gblob[rec + 4]), int(gblob[rec + 7])
        bad = []
        for word, value in [(0, 0), (1, 2), (3, len(gblob) + 4), (2, -1), (2, 100000), (rec + 0, -1), (rec + 1, 8),
                            (rec + 2, 1 << 20), (rec + 3, 0), (rec + 3, 17), (rec + 8, 5), (rec + 9, 1 << 20),
                            (role_off + 1, -1), (role_off + 2, 1 << 20), (role_off + 3, 4), (4, 1 << 20)]:
            b = gblob.copy()
            b[word] = value
            bad.append(b)
        if int(gblob[rec + 6]) > 0:
            b = gblob.copy()
            b[anchor_off] = topo.n
            bad.append(b)
        for b in bad:
            c1 = _code(lambda: eng.place_groups(b))
            c2 = _code(lambda: eng.place_groups_committed(b))
            assert c1 == c2 and c1 != 0, (c1, c2)
        again = eng.place_groups_committed(gblob)
        assert all(np.array_equal(x, y) for x, y in zip(again[:3], good[:3]))
    finally:
        eng.close()


def test_tables_beyond_shared_memory_return_elimit():
    from test_gpu_groups_limits import _build as build_limits, _one_role_groups, _wide_group
    n = 4097
    rng = np.random.default_rng(120)
    topo = synth.make_topology(n, seed=3, tiers=4, max_free=4)
    wide = _wide_group(rng, 16, 5, n)
    p = np.asarray(wide.pair)
    p[:, 15] = 0
    wide.pair = p.tolist()
    nodes = rng.choice(n, size=120, replace=False)
    wide.anchors = [(int(x), 15, 1) for x in nodes]
    groups = _one_role_groups(rng, 20, 10, n)
    groups.insert(3, wide)
    gblob = build_limits(groups)
    eng = engine(topo)
    try:
        with pytest.raises(RbgTopoError) as e:
            eng.place_groups_committed(gblob)
        assert e.value.code == -6 and "per-wave fallback" in str(e.value)
        small = build_limits(groups[:3] + groups[4:])
        check(eng, topo, small)
    finally:
        eng.close()


def test_snapshot_calls_unchanged_around_committed_calls():
    case = gg.make_case(5, 2049)
    eng = engine(case.topo)
    try:
        def snapshot_results():
            a, s, d = eng.place_groups(case.blob)
            h = eng.stage_groups(case.blob)
            try:
                eng.run_staged(h, 1)
                fa, fs, fd = eng.fetch(h)
            finally:
                eng.release(h)
            return [x.copy() for x in (a, s, d, fa, fs, fd)]
        before = snapshot_results()
        eng.place_groups_committed(case.blob)
        eng.place_groups_committed(case.blob)
        after = snapshot_results()
        assert all(np.array_equal(x, y) for x, y in zip(before, after))
    finally:
        eng.close()
