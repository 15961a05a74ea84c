"""GPU: whole-group placement (rbgtopo_place_groups, rbgtopo_stage_groups) at the limits of the GROUPS ABI against
the oracle's wave loop run on the very same raw GROUPS blob (oracle.wave_loop.groups_from_blob).

The plugin's fleets never leave 3 role rows per wave, 0/1 symmetric pair matrices, demand 0/1 and node counts that
are multiples of 4.  The fleets here come from tests/groups_gen.py: 8-role waves (256-thread CTAs of k_plan_group),
16-role groups, weighted asymmetric pairs, ragged node counts (the tail mask of k_emit_rows), per-wave and global-list
fallbacks, and scores at the edge of the exactness bound."""
import os

import numpy as np
import pytest

import groups_gen as gg
from oracle import wave_loop
from rbg_b200 import synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, Group, GroupsBuilder
from rbg_b200.engine import plan_steps

pytestmark = pytest.mark.gpu


def oracle_plan(topo, gblob):
    """The oracle's wave loop on a GROUPS blob: (states, per wave (wave, group indices, oracle result))."""
    groups = wave_loop.groups_from_blob(gblob)
    index = {id(g): i for i, g in enumerate(groups)}
    waves = []
    states, _ = wave_loop.run_fleet(topo, groups, want_matrix=True, want_topk=True,
                                    on_wave=lambda w, act, blob, r: waves.append((w, [index[id(s.g)] for s in act], r)))
    return states, waves


def group_slices(states):
    out, off = [], 0
    for st in states:
        n = sum(st.pending)
        out.append(slice(off, off + n))
        off += n
    return out


def check_direct(eng, states, gblob):
    """place_groups (direct path by default): placements, status and domain of every group, status-1 groups included
    (the library re-runs them through its host loop)."""
    a, s, d = eng.place_groups(gblob)
    for i, (st, sl) in enumerate(zip(states, group_slices(states))):
        res = st.result()
        assert a[sl].tolist() == st.assign_in_group_order(), ("direct", i)
        assert (int(s[i]), int(d[i])) == (res["status"], res["domain"]), ("direct", i, int(s[i]), int(d[i]), res["status"], res["domain"])


def check_staged(eng, topo, states, waves, gblob):
    """stage_groups -> run_staged -> fetch: dense-matrix bits of every row and the top-K keys of every role row for
    every wave the oracle ran (a group that lost a replica only up to that wave: later waves use the predicted need),
    placements of status 0 / 2 groups, status 1 reported as such."""
    h = eng.stage_groups(gblob)
    try:
        eng.run_staged(h, 1)
        return check_handle(eng, topo, states, waves, gblob, h)
    finally:
        eng.release(h)


def defined_rows(topo, states, waves, gblob):
    """The replica rows and role rows whose content a pass defines, i.e. those check_handle compares: every wave the
    oracle ran, a group that lost a replica only up to that wave (later waves of it are not selected)."""
    first = {(int(st[0]), int(st[1])): (int(st[4]), int(st[5])) for st in plan_steps(gblob, topo.n, len(topo.domain_owner))}
    lost, rows, roles = set(), [], []
    for w, gis, r in waves:
        off = 0
        for gi in gis:
            wave = states[gi].waves[w]
            cnt = sum(c for _, _, c in wave)
            if gi not in lost:
                row0, role0 = first[(gi, w)]
                rows += range(row0, row0 + cnt)
                roles += range(role0, role0 + len(wave))
                if (r["assign"][off:off + cnt] < 0).any():
                    lost.add(gi)
            off += cnt
    return rows, roles


def check_handle(eng, topo, states, waves, gblob, h):
    """The checks of check_staged on a handle whose last pass has been enqueued; returns the rows compared."""
    a, s, d = eng.fetch(h)
    first = {(int(st[0]), int(st[1])): (int(st[4]), int(st[5])) for st in plan_steps(gblob, topo.n, len(topo.domain_owner))}
    lost = set()
    rows = 0
    for w, gis, r in waves:
        off = rr = 0
        for k, gi in enumerate(gis):
            wave = states[gi].waves[w]
            cnt, P = sum(c for _, _, c in wave), len(wave)
            if gi not in lost:
                row0, role0 = first[(gi, w)]
                for j in range(cnt):
                    got, exp = eng.read_scores(h, row0 + j), r["matrix"][off + j]
                    bad = np.nonzero(got.view(np.uint32) != exp.view(np.uint32))[0]
                    assert len(bad) == 0, ("row", w, gi, j, len(bad), int(bad[0]), float(got[bad[0]]), float(exp[bad[0]]))
                for p in range(P):
                    got = eng.read_topk(h, role0 + p, 32)
                    assert np.array_equal(got, r["topk"][rr + p]), ("topk", w, gi, p, got[:6], r["topk"][rr + p][:6])
                rows += cnt
                if (r["assign"][off:off + cnt] < 0).any():
                    lost.add(gi)
            off += cnt
            rr += P
    for i, (st, sl) in enumerate(zip(states, group_slices(states))):
        res = st.result()
        if res["status"] == 1:
            assert int(s[i]) == 1, ("staged", i)
            continue
        assert a[sl].tolist() == st.assign_in_group_order(), ("staged", i)
        assert (int(s[i]), int(d[i])) == (res["status"], res["domain"]), ("staged", i)
    return rows


def pending_groups(gblob):
    return sum(1 for g in range(int(gblob[2])) if int(gblob[8 + 12 * g + 9]) > 0)


def plan_ran(eng, gblob, direct=False):
    """k_plan_group ran with one CTA per group with pending replicas (the per-wave fallback when forced).  With
    RBGTOPO_SPLIT_MIN_GROUPS place_groups launches it once per half of the fleet and the count is the last half's."""
    want = 0 if os.environ.get("RBGTOPO_PER_WAVE_PLAN") else pending_groups(gblob)
    got = eng.stats()["plan_ctas"]
    if direct and want and os.environ.get("RBGTOPO_SPLIT_MIN_GROUPS"):
        assert 0 < got <= want, (eng.stats(), want)
    else:
        assert got == want, (eng.stats(), want)


@pytest.mark.parametrize("seed,n,scarce,excl", gg.CASES)
def test_generated_fleets_match_oracle(seed, n, scarce, excl):
    from gpu_util import new_engine
    case = gg.make_case(seed, n, scarce=scarce, exclusive=excl)
    states, waves = oracle_plan(case.topo, case.blob)
    eng = new_engine(case.topo)
    try:
        check_direct(eng, states, case.blob)
        plan_ran(eng, case.blob, direct=True)
        assert check_staged(eng, case.topo, states, waves, case.blob) > 0
        plan_ran(eng, case.blob)
    finally:
        eng.close()


def test_chunked_node_axis():
    """chunk_nodes = 128 at N = 4097: 33 chunks per row, the last one a single ragged node."""
    from gpu_util import new_engine
    case = gg.make_case(11, 4097)
    states, waves = oracle_plan(case.topo, case.blob)
    eng = new_engine(case.topo, chunk_nodes=128)
    try:
        check_direct(eng, states, case.blob)
        check_staged(eng, case.topo, states, waves, case.blob)
    finally:
        eng.close()


def _one_role_groups(rng, n_groups, gid0, n_nodes):
    out = []
    for g in range(n_groups):
        anchors = [(int(rng.integers(0, n_nodes)), 0, int(rng.integers(1, 3)))] if g % 3 == 0 else []
        out.append(Group(gid=gid0 + g, roles=[(0, int(rng.integers(1, 6)), int(rng.integers(0, 3)), ROLE_EXCLUSIVE)],
                         pair=[[int(rng.integers(0, 4))]], anchors=anchors, flags=STEP_EXCLUSIVE if g % 4 == 1 else 0))
    return out


def _build(groups):
    gb = GroupsBuilder()
    for g in groups:
        gb.add(g)
    return gb.build()


def _wide_group(rng, q, gid, n_nodes):
    """q roles in one level, 1-3 pending each: waves of 8 role rows."""
    p = rng.integers(0, 4, size=(q, q))
    np.fill_diagonal(p, 0)
    return Group(gid=gid, roles=[(0, int(rng.integers(1, 4)), int(rng.integers(0, 3)), ROLE_EXCLUSIVE) for _ in range(q)],
                 pair=p.tolist(), anchors=[(int(rng.integers(0, n_nodes)), int(rng.integers(0, q)), 2)])


@pytest.mark.parametrize("q", [16, 8])
def test_one_wide_group_among_one_role_groups(q):
    """QB = 16 (or one 8-role wave) while most groups have Q = 1: the batch geometry is set by one group."""
    from gpu_util import new_engine
    n = 2049
    rng = np.random.default_rng(q)
    topo = synth.make_topology(n, seed=q, tiers=3, owned_frac=0.2, max_free=4)
    groups = _one_role_groups(rng, 40, 10, n)
    groups.insert(17, _wide_group(rng, q, 5, n))
    gblob = _build(groups)
    states, waves = oracle_plan(topo, gblob)
    assert max(len(w) for st in states for w in st.waves) == 8
    eng = new_engine(topo)
    try:
        check_direct(eng, states, gblob)
        plan_ran(eng, gblob, direct=True)
        check_staged(eng, topo, states, waves, gblob)
        plan_ran(eng, gblob)
    finally:
        eng.close()


def _place_geom(gblob, topo, wsum):
    import ctypes as C
    from rbg_b200 import _lib
    lib = _lib.load()
    gb = np.ascontiguousarray(gblob, dtype=np.int32)
    degp1 = (np.diff(topo.row_ptr) + 1).astype(np.int32)
    order = np.zeros(max(1, int(gb[2])), dtype=np.int32)
    geom = np.zeros(8, dtype=np.int32)
    i32 = _lib.i32p
    rc = lib.rbgtopo_place_describe(gb.ctypes.data_as(i32), len(gb), topo.n, len(topo.domain_owner), degp1.ctypes.data_as(i32),
                                    wsum, order.ctypes.data_as(i32), len(order), geom.ctypes.data_as(i32))
    assert rc == 0
    return geom


@pytest.mark.parametrize("n_anchor_nodes", [120, 2000])
def test_tables_beyond_shared_memory_take_the_per_wave_path(n_anchor_nodes):
    """A 16-role group with scheduled pods on many distinct nodes: its table of patched nodes does not fit k_plan_group's
    shared memory (200 KB), so the plan runs one launch per wave; with ~2 000 pods not even one step's patched set fits
    the shared-memory selection and the global candidate list (k_select_assign) takes over.  The scheduled pods of the
    heavy role have pair weight 0 toward the pending roles (keeps the exactness bound), a few weighted ones do not."""
    from gpu_util import new_engine
    n = 4097
    rng = np.random.default_rng(n_anchor_nodes)
    topo = synth.make_topology(n, seed=3, tiers=4, max_free=4)
    wide = _wide_group(rng, 16, 5, n)
    p = np.asarray(wide.pair)
    p[:, 15] = 0
    wide.pair = p.tolist()
    nodes = rng.choice(n, size=n_anchor_nodes, replace=False)
    wide.anchors = [(int(x), 15, 1) for x in nodes] + [(int(x), int(rng.integers(0, 15)), 2) for x in nodes[:12]]
    groups = _one_role_groups(rng, 20, 10, n)
    groups.insert(3, wide)
    gblob = _build(groups)
    wsum = gg.wsum_max(topo)
    assert gg.exact_ok(wide, wsum)
    geom = _place_geom(gblob, topo, wsum)
    cap = int(geom[4])
    ht = 64
    while ht <= cap:
        ht <<= 1
    assert ht * 4 * (2 + 16) + cap * 16 > 250 * 1024, cap          # k_plan_group's table + dense view alone
    states, waves = oracle_plan(topo, gblob)
    eng = new_engine(topo)
    try:
        check_staged(eng, topo, states, waves, gblob)
        assert eng.stats()["plan_ctas"] == 0                 # fresh context: k_plan_group never launched
        check_direct(eng, states, gblob)
        if os.environ.get("RBGTOPO_SPLIT_MIN_GROUPS"):   # the half without the wide group still fits k_plan_group
            assert eng.stats()["plan_ctas"] < pending_groups(gblob)
        else:
            assert eng.stats()["plan_ctas"] == 0
    finally:
        eng.close()


def test_exactness_edge():
    """tiers = 1: every row sums to 7 000, so a step is admitted while (7 000 + 8 000) x (need·8 + Σ pair·count) < 2^24,
    i.e. need·8 + Σ pair·count <= 1 118.  Role 0 has need 2 (the pending replicas of role 1) and 1 102 scheduled pods of
    role 1 in repeated records: 16 + 1 102 = 1 118, scores up to ~8.9e6 (the top binade of exact fp32 integers) and bit
    parity.  One more pod is -4 on the direct and on the staged path."""
    from gpu_util import new_engine
    from rbg_b200.engine import RbgTopoError
    n = 64
    topo = synth.make_topology(n, seed=5, tiers=1, max_free=4)
    assert gg.wsum_max(topo) == 7000

    m = int(np.nonzero(topo.free > 0)[0][0])          # the heavy pods sit on a node that stays feasible

    def blob(extra):
        g = Group(gid=1, roles=[(0, 1, 1, ROLE_EXCLUSIVE), (1, 2, 1, ROLE_EXCLUSIVE)], pair=[[0, 1], [1, 0]],
                  anchors=[(m, 1, 600), (m, 1, 502 + extra), (12, 0, 1)])
        return _build([g, Group(gid=2, roles=[(0, 3, 1, ROLE_EXCLUSIVE)], pair=[[1]], anchors=[(40, 0, 1)])])

    ok, bad = blob(0), blob(1)
    states, waves = oracle_plan(topo, ok)
    top = max(float(r["matrix"].max()) for _, _, r in waves)
    assert 2 ** 23 <= top < 2 ** 24, top
    eng = new_engine(topo)
    try:
        check_direct(eng, states, ok)
        check_staged(eng, topo, states, waves, ok)
        for f in (eng.place_groups, eng.stage_groups):
            with pytest.raises(RbgTopoError) as ei:
                f(bad)
            assert ei.value.code == -4, str(ei.value)
        check_direct(eng, states, ok)   # the context is unharmed
    finally:
        eng.close()
