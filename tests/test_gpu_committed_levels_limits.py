"""GPU: committed batches at exclusive levels at their limits (DESIGN.md §3.8 / §3.9, the <true> instantiations of
k_plan_group_commit / k_commit_claims / k_commit_diff), bit for bit against committed_levels_oracle on the cases of
tests/commit_levels_limits_cases.py: assign, status, domain, exactly G rounds on the chains, the committed-ranked call
(n_alt 0, 1 and 8) against committed_alternates_oracle, and invariants read from the outputs alone (capacity, the
reference's anti-affinity terms, one gid per reported domain and level unless fixed).  Also: moved non-exclusive groups
equal to the level-0 batch, world 2 and 4, refreshes while a ~200-round level call runs, the shared-memory ceiling on
the <true> path, and N = 2^20 + 1 with seven installed levels."""
import copy
import resource
import threading
import time

import numpy as np
import pytest

import commit_levels_gen as clg
import commit_levels_limits_cases as cl
import committed_alternates_oracle as cao
import levels_limits_cases as llc
from committed_levels_oracle import group_levels
from gpu_util import new_engine
from oracle import wave_loop
from rbg_b200 import synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, STEP_GANG, Group
from rbg_b200.engine import RbgTopoError

pytestmark = pytest.mark.gpu

CASES = cl.cases()


def engine(c, **kw):
    eng = new_engine(c.topo, committed_levels=True, **kw)
    eng.set_exclusive_levels(c.lv[1:], c.occ, level_n_domains=c.nd[1:])
    return eng


def pending_groups(gblob):
    return sum(1 for g in range(int(gblob[2])) if int(gblob[8 + 12 * g + 9]) > 0)


def same(x, y):
    return all(np.array_equal(np.asarray(p), np.asarray(q)) for p, q in zip(x[:3], y[:3]))


def invariants(c, a, s, d, brute_force=True):
    """No node asked for more than free; no anti-affinity term broken (brute force over every record: skipped at a
    million nodes and 610 000 records, where the oracle comparison alone stands); two gids report one (level, domain)
    only where one of them was fixed to it."""
    groups = c.extra["groups"]
    used = np.zeros(c.topo.n, np.int64)
    off = 0
    for g, og in enumerate(wave_loop.groups_from_blob(c.blob)):
        st = wave_loop.GroupState(og)
        for ri in st.order:
            for _ in range(st.pending[ri]):
                if a[off] >= 0 and s[g] != 2:
                    used[a[off]] += og.roles[ri].demand
                off += 1
    assert (used <= c.topo.free).all(), np.nonzero(used > c.topo.free)[0][:8]
    if brute_force:
        assert clg.violations(c.lv, c.occ, c.blob, a, s) == []
    rep = {}
    for g, grp in enumerate(groups):
        if grp.flags & STEP_EXCLUSIVE and d[g] >= 0 and s[g] != 2:
            rep.setdefault((grp.level, int(d[g])), []).append((grp.gid, grp.fixed_domain >= 0))
    for k, v in rep.items():
        if len({gid for gid, _ in v}) > 1:
            assert any(fx for _, fx in v), (k, v)


def check(eng, c, brute_force=True):
    got = eng.place_groups_committed(c.blob)
    a, s, d, rounds = got
    ea, es, ed = cl.expected(c)
    assert np.array_equal(a, ea), (c.name, np.nonzero(a != ea)[0][:8])
    assert np.array_equal(s, es), (c.name, np.nonzero(s != es)[0][:8])
    assert np.array_equal(d, ed), (c.name, np.nonzero(d != ed)[0][:8])
    if c.rounds is not None:
        assert rounds == c.rounds, (c.name, rounds, c.rounds)
    else:
        assert 1 <= rounds <= pending_groups(c.blob), (c.name, rounds)
    invariants(c, a, s, d, brute_force)
    return got


def check_ranked(eng, c, got):
    owner = cl.owner(c)
    exp = cao.run_fleet_committed_ranked(c.topo, wave_loop.groups_from_blob(c.blob), 8, fast=True,
                                         levels=dict(group_levels=group_levels(c.blob), level_domain=c.lv,
                                                     owner=owner, n_domains=c.nd))
    for F in (0, 1, 8):
        r = eng.place_groups_committed_ranked(c.blob, F)
        assert same(r, got) and r[3] == got[3], (c.name, F)
        sc, an, asc = (np.asarray(x) for x in r[4:])
        assert np.array_equal(sc.view(np.uint32), exp[3].view(np.uint32)), (c.name, F)
        assert an.size == asc.size == F * len(sc), (c.name, F)
        if F:
            assert np.array_equal(an.reshape(-1, F), exp[4][:, :F]), (c.name, F)
            assert np.array_equal(asc.reshape(-1, F).view(np.uint32),
                                  np.ascontiguousarray(exp[5][:, :F]).view(np.uint32)), (c.name, F)


@pytest.mark.parametrize("i", range(len(CASES)), ids=[c.name for c in CASES])
def test_cases_match_the_oracle_plain_and_ranked(i):
    c = CASES[i]
    eng = engine(c)
    try:
        got = check(eng, c)
        check_ranked(eng, c, got)
    finally:
        eng.close()


def test_true_path_equals_the_level0_batch():
    """Non-exclusive groups moved to levels >= 1 (the <true> kernels, lmask within {0}): the same outputs and rounds
    as the unmoved batch (the <false> kernels) on the same ctx, and the oracle's."""
    for base, moved in cl.level0_pairs():
        eng = engine(base)
        try:
            r0 = check(eng, base)
            r1 = check(eng, moved)
            assert same(r0, r1) and r0[3] == r1[3], base.name
        finally:
            eng.close()


@pytest.mark.parametrize("world", [2, 4])
def test_world_contexts_equal_world_1(world):
    for c in [cl.chain(64, "P"), cl.chain(64, "mix"), cl.offsets()]:
        e1 = engine(c)
        try:
            ref = check(e1, c)
        finally:
            e1.close()
        engs = [engine(c, rank=r, world=world) for r in range(world)]
        try:
            for r, e in enumerate(engs):
                got = e.place_groups_committed(c.blob)
                assert same(got, ref) and got[3] == ref[3], (c.name, r)
        finally:
            for e in engs:
                e.close()


def _refreshed(c, kind):
    """(the refresh as a call on an engine, the case it installs).  Each one flips the chain's first link: a_0 loses
    its room (free), a record of another gid blocks it (records only), or the links' partitions go (reinstall)."""
    a0 = c.extra["a"][0]
    if kind == "free":
        free = c.topo.free.copy()
        free[a0] = 0
        t = synth.Topology(c.topo.row_ptr, c.topo.col_idx, c.topo.edge_w, free, c.topo.domain, c.topo.domain_owner)
        return (lambda e: e.update_nodes(free=free)), cl.Case(c.name, t, c.lv, c.nd, c.occ, c.blob, extra=c.extra)
    if kind == "records":
        occ = np.array([[a0, 99, 1]], np.int32)
        return (lambda e: e.set_exclusive_levels(None, occ)), cl.Case(c.name, c.topo, c.lv, c.nd, occ, c.blob,
                                                                       extra=c.extra)
    lv = np.stack([c.lv[0]] + [np.arange(c.topo.n)] * 7).astype(np.int32)
    nd = [c.nd[0]] + [c.topo.n] * 7
    return ((lambda e: e.set_exclusive_levels(lv[1:], c.occ, level_n_domains=nd[1:])),
            cl.Case(c.name, c.topo, lv, nd, c.occ, c.blob, extra=c.extra))


@pytest.mark.parametrize("kind", ["free", "records", "partitions"])
def test_a_refresh_during_a_level_call_lands_between_calls(kind, record_property):
    """The ~200-round chain at all eight levels in one thread, a refresh issued 2 ms into the call from another: the
    call returns the oracle's result on one snapshot, never a mix, and the next call places on the new one."""
    c = cl.chain(*cl.REFRESH_CHAIN)
    refresh, new_c = _refreshed(c, kind)
    old, new = cl.expected(c), cl.expected(new_c)
    assert not same(old, new)
    eng = engine(c)
    try:
        out = {}
        started = threading.Event()

        def call():
            started.set()
            t0 = time.perf_counter()
            out["r"] = eng.place_groups_committed(c.blob)
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
            assert r[3] == cl.REFRESH_CHAIN[0]
        again = eng.place_groups_committed(c.blob)
        assert same(again, new)
    finally:
        eng.close()


def test_tables_on_both_sides_of_the_shared_memory_ceiling_at_a_level():
    """A 16-role exclusive group at level 6 whose table of patched nodes is the largest that fits shared memory is
    placed like the oracle; one more anchored node and the call returns RBGTOPO_ELIMIT, the ctx still usable."""
    from test_gpu_groups_limits import _one_role_groups, _wide_group
    n = 4097
    rng = np.random.default_rng(131)
    topo = synth.make_topology(n, seed=3, tiers=4, max_free=4)
    topo.domain_owner[:] = -1
    wide = _wide_group(rng, 16, 5, n)
    p = np.asarray(wide.pair)
    p[:, 15] = 0
    wide.pair = p.tolist()
    wide.flags, wide.level = STEP_EXCLUSIVE, 6
    nodes = rng.permutation(n)
    others = _one_role_groups(rng, 12, 10, n)
    for k, g in enumerate(others):
        g.level = 4 + k % 4
    lv, nd = llc.partitions47(topo, 131, "random")

    def case(k):
        wide.anchors = [(int(x), 15, 1) for x in nodes[:k]]
        gr = [copy.copy(g) for g in others[:3] + [wide] + others[3:]]
        return cl.Case(f"ceiling{k}", topo, lv, nd, np.zeros((0, 3), np.int32), cl._blob(gr), extra=dict(groups=gr))
    eng = engine(case(0))
    try:
        def fits(k):
            try:
                eng.place_groups_committed(case(k).blob)
                return True
            except RbgTopoError as e:
                assert e.code == -6, e
                return False
        lo_k, hi_k = 0, 1
        while fits(hi_k):
            lo_k, hi_k = hi_k, 2 * hi_k
        while hi_k - lo_k > 1:
            mid = (lo_k + hi_k) // 2
            lo_k, hi_k = (mid, hi_k) if fits(mid) else (lo_k, mid)
        assert lo_k > 0
        with pytest.raises(RbgTopoError) as e:
            eng.place_groups_committed(case(lo_k + 1).blob)
        assert e.value.code == -6 and "shared memory" in str(e.value)
        check(eng, case(lo_k))
    finally:
        eng.close()


def million(n=llc.FULL_N):
    """llc.derivation's seven levels and ~7.4 M domains; 24 groups over all eight levels racing for the head of the
    background order (a short chain of claims), shared gids, gangs."""
    d = llc.derivation(n)
    groups = []
    for k in range(24):
        groups.append(Group(gid=6000 + k % 20, roles=[(0, 1 + k % 3, 1, ROLE_EXCLUSIVE)], pair=[[1]],
                            flags=STEP_EXCLUSIVE | (STEP_GANG if k % 5 == 4 else 0), level=k % 8))
    return cl.Case(f"million/{n}", d.topo, d.lv, d.nd, d.occ, cl._blob(groups), extra=dict(groups=groups))


def test_a_million_nodes_at_seven_levels(capsys):
    c = million()
    assert sum(c.nd) > 7_000_000 and c.lv.shape[0] == 8
    t0 = time.perf_counter()
    eng = engine(c)
    try:
        got = check(eng, c, brute_force=False)
    finally:
        eng.close()
    wall = time.perf_counter() - t0
    rss = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1024
    with capsys.disabled():
        print(f"\nmillion-node committed level batch: rounds {got[3]}, wall {wall:.1f} s (install, call and oracle), "
              f"peak host RSS {rss:.0f} MiB")
