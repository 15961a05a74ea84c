"""GPU: the per-snapshot vectors every score and top-K list is built on — base = W·min(free, 8), the background order
(compact-key radix sort, order_all when world > 1) and pos, its inverse, kept by the incremental repair — read back with
rbgtopo_read_snapshot and compared word for word with the plain references of tests/topo_gen.py, on the irregular
snapshots of that generator: hub rows around k_base's staging limit, isolated rows and runs of them, large-scale ties,
the largest base the compact key reserves bits for, N past the fmin staging limit, and inexact snapshots.  Placements on
the same snapshots are checked against the oracle, and the delta repair against a mirror of free[] after every call."""
import os

import numpy as np
import pytest

import topo_gen as tg
from gpu_util import check_batch, new_engine
from oracle import placer as oracle_placer
from rbg_b200.blob import ROLE_EXCLUSIVE, BlobBuilder, Group, GroupsBuilder, Step
from rbg_b200.engine import RbgTopoError, TopoPlacer

pytestmark = pytest.mark.gpu

DELTA_MAX_AFFECTED = 2048
NO_DELTA = bool(os.environ.get("RBGTOPO_NO_DELTA"))


def check_snapshot(eng, topo, world1=True):
    """base bit for bit, order word for word, pos (world 1) against the references of topo.free."""
    base = eng.read_snapshot("base")
    lo, hi = eng.slab()
    if tg.exact_snapshot(topo):
        exp = tg.base_ref(topo)
        bad = np.nonzero(base.view(np.uint32) != exp.view(np.uint32))[0]
        assert len(bad) == 0, ("base", len(bad), int(bad[0]), float(base[bad[0]]), float(exp[bad[0]]))
    else:
        exp = base                                     # inexact: the order must follow the device's own bits
    order = eng.read_snapshot("order")
    ref = tg.order_ref(exp, lo, hi)
    if not np.array_equal(order, ref):
        bad = np.nonzero(order != ref)[0]
        raise AssertionError(("order", len(bad), int(bad[0]), int(tg.key_node(order[bad[:1]])[0]),
                              int(tg.key_node(ref[bad[:1]])[0])))
    assert np.array_equal(eng.read_snapshot("order_all"), tg.order_ref(exp)), "order_all"
    if world1:
        assert np.array_equal(eng.read_snapshot("pos"), tg.pos_ref(ref)), "pos"


def repairs(eng):
    return int(eng.read_snapshot("delta_repairs")[0])


def est_of(topo, nodes):
    u = np.unique(nodes)
    return int((np.diff(topo.row_ptr)[u] + 1).sum())


def delta(eng, topo, nodes, vals, check=True):
    """update_nodes_delta + the mirror; asserts the repair counter moved iff the library should have repaired."""
    nodes = np.asarray(nodes, dtype=np.int32)
    vals = np.asarray(vals, dtype=np.int32)
    before = repairs(eng)
    eng.update_nodes_delta(nodes, vals)
    for nd, v in zip(nodes, vals):
        topo.free[nd] = v
    want = int(est_of(topo, nodes) <= DELTA_MAX_AFFECTED and not NO_DELTA and eng.world == 1 and len(nodes) > 0)
    if check:
        assert repairs(eng) - before == want, (repairs(eng) - before, want, est_of(topo, nodes))
        check_snapshot(eng, topo, eng.world == 1)
    return want


# ---------------------------------------------------------------- snapshot after set_topology / update_nodes
@pytest.mark.parametrize("name", tg.NAMES)
def test_snapshot_after_set_topology_and_update_nodes(name):
    topo = tg.copy_topo(tg.make(name).topo)
    rng = np.random.default_rng(len(name))
    eng = new_engine(topo)
    try:
        check_snapshot(eng, topo)
        assert repairs(eng) == 0
        free = topo.free.copy()
        flip = rng.random(topo.n) < 0.3
        free[flip] = rng.choice([0, 3, 8, 9, 12, tg.MAX_FREE], size=int(flip.sum()))
        if not tg.exact_snapshot(topo):
            free[np.argmax(tg.wsum_rows(topo))] = 30       # the hub keeps its neighbourhood's base past 2^24
        owner = topo.domain_owner.copy()
        owner[rng.random(len(owner)) < 0.2] = 77
        topo.free = free.astype(np.int32)
        eng.update_nodes(topo.free, owner)
        topo.domain_owner = owner
        check_snapshot(eng, topo)
    finally:
        eng.close()


# ---------------------------------------------------------------- inexact snapshots
@pytest.mark.parametrize("name", [n for n in tg.NAMES if tg.BUILDERS[n][0] == "inexact"])
def test_inexact_snapshot_admits_need_0_only(name):
    topo = tg.copy_topo(tg.make(name).topo)
    eng = new_engine(topo)
    try:
        check_snapshot(eng, topo)                          # a permutation, sorted by the device's own base bits
        base = eng.read_snapshot("base")
        assert float(base.max()) >= 2 ** 24
        hub = int(np.argmax(tg.wsum_rows(topo)))
        assert base[hub] == tg.k_base_fp32(topo, hub)
        bad = BlobBuilder().add(Step(gid=0, roles=[(2, 1, 1, 0)], pair=[])).build()
        with pytest.raises(RbgTopoError) as ei:
            eng.score_assign(bad)
        assert ei.value.code == -4
        g = GroupsBuilder().add(Group(gid=1, roles=[(0, 2, 1, ROLE_EXCLUSIVE)], pair=[[1]])).build()
        with pytest.raises(RbgTopoError) as ei:
            eng.place_groups(g)
        assert ei.value.code == -4
        row_w = tg.wsum_max(topo) + tg.SELF_W
        lim = -(-(1 << 24) // row_w) - 1                  # largest anchor mass the exactness check admits
        nbr = int(topo.col_idx[topo.row_ptr[hub]])
        if lim >= 4:                                       # anchor mass 1 + 3 <= lim
            anc, pair = [(hub, 0, 1), (nbr, 1, 3)], [[1, 1]]
        else:                                              # no mass at all: pair weight 0
            anc, pair = [(hub, 1, 2)], [[0, 0]]
        bb = BlobBuilder()
        for s in range(6):
            bb.add(Step(gid=s, roles=[(1 + s % 4, s % 3, 0, 0)], pair=pair, anchors=anc))
        check_batch(eng, topo, bb.build())
    finally:
        eng.close()


# ---------------------------------------------------------------- world 2 / 4 on one device
def _ties100():
    return tg.ties(100, "zero", 1)


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("name", ["ties100", "sparse_255", "sparse_257", "large_131073"])
def test_sharded_snapshot(world, name):
    topo = _ties100() if name == "ties100" else tg.make(name).topo
    engs = []
    try:
        for r in range(world):
            e = TopoPlacer(device=0, rank=r, world=world)
            e.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
            engs.append(e)
        slabs = [e.slab() for e in engs]
        assert slabs[0][0] == 0 and slabs[-1][1] == topo.n and all(a[1] == b[0] for a, b in zip(slabs, slabs[1:]))
        assert all(lo % 128 == 0 for lo, _ in slabs)
        if topo.n < 256:
            assert any(lo == hi for lo, hi in slabs)    # empty slabs
        for e in engs:
            check_snapshot(e, topo, world1=False)
            with pytest.raises(RbgTopoError):
                e.read_snapshot("pos")
    finally:
        for e in engs:
            e.close()


# ---------------------------------------------------------------- placements on the same snapshots
def _hubs_and_isolated(topo, k=4):
    deg = np.diff(topo.row_ptr)
    return np.argsort(-deg, kind="stable")[:k].tolist(), np.nonzero(deg == 0)[0][:k].tolist()


def _steps(topo, seed, n_steps=10):
    """Demands {0, 1, 2, 8, 9, 12}, need 1..16, anchors on hubs and isolated nodes, inside the exactness bound."""
    rng = np.random.default_rng(seed)
    hubs, iso = _hubs_and_isolated(topo)
    row_w = tg.wsum_max(topo) + tg.SELF_W
    lim = -(-(1 << 24) // row_w) - 1
    bb = BlobBuilder()
    for s in range(n_steps):
        P = int(rng.integers(1, 4))
        Q = P + 1
        need_max = max(1, min(16, lim // 8))
        roles = [(int(rng.integers(1, 7)), int(rng.choice([0, 1, 2, 8, 9, 12])), int(rng.integers(1, need_max + 1)), ROLE_EXCLUSIVE)
                 for _ in range(P)]
        anc = [(int(rng.choice(hubs + iso)), int(rng.integers(0, Q)), int(rng.integers(1, 3))) for _ in range(int(rng.integers(0, 5)))]
        pair = rng.integers(0, 3, size=(P, Q))
        for p in range(P):
            while roles[p][2] * 8 + sum(int(pair[p][q]) * c for _, q, c in anc) > lim:
                if pair[p].any():
                    pair[p][int(np.argmax(pair[p]))] -= 1
                else:
                    roles[p] = roles[p][:2] + (roles[p][2] - 1, roles[p][3])
        bb.add(Step(gid=s, roles=roles, pair=pair.tolist(), anchors=anc, consumed=[(int(rng.integers(0, topo.n)), 1)]))
    return bb.build()


def _fleet(topo, seed):
    from test_gpu_groups_limits import _build, _one_role_groups, _wide_group
    import groups_gen as gg
    rng = np.random.default_rng(seed)
    groups = _one_role_groups(rng, 12, 10, topo.n)
    groups.insert(5, _wide_group(rng, 16, 5, topo.n))
    hubs, iso = _hubs_and_isolated(topo)
    groups[5].anchors += [(hubs[0], 1, 1)] + ([(iso[0], 2, 1)] if iso else [])
    for g in groups:
        while not gg.exact_ok(g, tg.wsum_max(topo)):
            p = np.asarray(g.pair)
            p[np.unravel_index(int(np.argmax(p)), p.shape)] -= 1
            g.pair = p.tolist()
    return _build(groups)


@pytest.mark.parametrize("name", ["hubs", "big_hub", "sparse_700", "sparse_129", "ties_ring", "maxbase_bits", "maxbase_2p24",
                                  "large_131072"])
def test_placement_parity(name):
    from test_gpu_groups_limits import check_direct, check_staged, oracle_plan
    topo = tg.copy_topo(tg.make(name).topo)
    eng = new_engine(topo)
    try:
        check_batch(eng, topo, _steps(topo, 1), check_matrix=topo.n < 100000)
        # scarce: most nodes full, the background walk goes deep into the order
        rng = np.random.default_rng(2)
        topo.free = np.where(rng.random(topo.n) < 0.85, 0, topo.free).astype(np.int32)
        eng.update_nodes(topo.free)
        check_snapshot(eng, topo)
        check_batch(eng, topo, _steps(topo, 3), check_matrix=topo.n < 100000)
        if name in ("hubs", "sparse_700", "large_131072"):
            gblob = _fleet(topo, 4)
            states, waves = oracle_plan(topo, gblob)
            check_direct(eng, states, gblob)
            check_staged(eng, topo, states, waves, gblob)
    finally:
        eng.close()


# ---------------------------------------------------------------- delta repair
@pytest.mark.parametrize("name", ["hubs", "sparse_700", "ties_ring"])
def test_300_small_deltas(name):
    topo = tg.copy_topo(tg.make(name).topo)
    rng = np.random.default_rng(300)
    eng = new_engine(topo)
    deg = np.diff(topo.row_ptr)
    light = np.nonzero(deg < 200)[0]
    try:
        n_rep = 0
        for i in range(300):
            k = int(rng.integers(1, 5))
            nodes = rng.choice(light, size=k)                      # duplicates possible: the last value wins
            if i % 37 == 0:
                nodes[0] = int(np.argmax(deg))                     # a hub: falls back where deg + 1 > 2 048
            vals = rng.choice([0, 1, 4, 7, 8, 9, 30, tg.MAX_FREE], size=k)
            n_rep += delta(eng, topo, nodes, vals)
        assert n_rep > 250 or NO_DELTA
        for i in range(50):                                        # a run with no reads in between
            nodes = rng.choice(light, size=2, replace=False)
            delta(eng, topo, nodes, rng.integers(0, 13, size=2), check=False)
        check_snapshot(eng, topo)
        check_batch(eng, topo, _steps(topo, 5), check_matrix=False)
    finally:
        eng.close()


def _ring_and_isolated():
    """Nodes 0..2999 in a ring (weight 100, free 8), 3000..3999 isolated: closed neighbourhoods of known size."""
    u = np.arange(3000)
    return tg.from_edges(4000, u, (u + 1) % 3000, np.full(3000, 100), np.full(4000, 8))


def test_delta_at_the_affected_limit():
    topo = _ring_and_isolated()
    eng = new_engine(topo)
    try:
        ring = np.arange(0, 3000, 3)[:682]                        # disjoint closed neighbourhoods of 3 nodes: 2 046
        iso = np.arange(3000, 4000)
        nodes = np.concatenate([ring, iso[:2]])
        assert est_of(topo, nodes) == 2048
        assert delta(eng, topo, nodes, np.full(len(nodes), 3)) == (0 if NO_DELTA else 1)
        nodes = np.concatenate([ring, iso[2:5]])                  # 2 049: the full refresh
        assert est_of(topo, nodes) == 2049
        assert delta(eng, topo, nodes, np.full(len(nodes), 5)) == 0
        nodes = np.concatenate([ring + 1, iso[5:7]])              # 2 048 again, on the full refresh's pos
        assert delta(eng, topo, nodes, np.full(len(nodes), 1)) == (0 if NO_DELTA else 1)
        nodes = np.arange(1000, 1600)                             # overlapping neighbourhoods: est 1 800, 602 affected
        assert delta(eng, topo, nodes, np.full(len(nodes), 2)) == (0 if NO_DELTA else 1)
        # node 0 and N-1, an isolated node (self term only), a node set to the value it has, duplicates in one call
        delta(eng, topo, [0, 3999], [0, 7])
        delta(eng, topo, [3500], [2])
        delta(eng, topo, [2000, 2000, 17, 2000], [0, 6, int(topo.free[17]), 4])
        # ties with unaffected nodes: back to the common value of the untouched ring
        delta(eng, topo, np.arange(1000, 1600), np.full(600, 8))
        check_batch(eng, topo, _steps(topo, 6), check_matrix=False)
    finally:
        eng.close()


def test_capacity_above_f_without_a_base_change():
    """free 12 -> 30 000 -> 9 on the nodes with the largest base: min(free, 8) never changes, the capacity does, and a
    step of demand 10-12 has to see it."""
    topo = tg.copy_topo(tg.make("hubs").topo)
    eng = new_engine(topo)
    try:
        light = np.nonzero(np.diff(topo.row_ptr) < 200)[0]        # no hub: the repair path, not the fallback
        top = light[np.argsort(-tg.base_int(topo)[light], kind="stable")[:40]]
        for v in (12, 30000, 9):
            delta(eng, topo, top, np.full(len(top), v))
        bb = BlobBuilder()
        for s in range(4):
            bb.add(Step(gid=s, roles=[(8, 10 + s % 3, 1, ROLE_EXCLUSIVE), (4, 9, 2, ROLE_EXCLUSIVE)], pair=[[1, 0], [0, 1]]))
        ref = check_batch(eng, topo, bb.build(), check_matrix=False)
        assert (ref["assign"] >= 0).any()
    finally:
        eng.close()


def test_delta_across_full_refreshes_and_topology_changes():
    small = tg.copy_topo(tg.make("sparse_700").topo)
    eng = new_engine(small)
    rng = np.random.default_rng(8)
    try:
        delta(eng, small, [1, 2, 699], [8, 0, 5])
        small.free = rng.integers(0, 13, size=small.n).astype(np.int32)
        eng.update_nodes(small.free)
        check_snapshot(eng, small)
        owner = small.domain_owner.copy()
        owner[::3] = 5
        eng.update_nodes(None, owner)
        small.domain_owner = owner
        check_snapshot(eng, small)
        delta(eng, small, [10, 11, 12], [0, 9, 3])
        big = tg.copy_topo(tg.make("large_131073").topo)          # buffers grow, the refresh graph is captured again
        eng.set_topology(big.row_ptr, big.col_idx, big.edge_w, big.free, big.domain, big.domain_owner)
        assert repairs(eng) == 0
        check_snapshot(eng, big)
        light = np.nonzero(np.diff(big.row_ptr) < 50)[0]
        delta(eng, big, [int(light[0]), int(light[len(light) // 2]), int(light[-1])], [0, 12, 3])
        check_batch(eng, big, _steps(big, 9, 4), check_matrix=False)
        small = tg.copy_topo(tg.make("sparse_257").topo)
        eng.set_topology(small.row_ptr, small.col_idx, small.edge_w, small.free, small.domain, small.domain_owner)
        check_snapshot(eng, small)
        delta(eng, small, [0, 256, 100], [3, 3, 0])
        check_batch(eng, small, _steps(small, 10, 4))
    finally:
        eng.close()


def test_world2_delta_falls_back():
    topo = tg.copy_topo(tg.make("sparse_700").topo)
    engs = [TopoPlacer(device=0, rank=r, world=2) for r in range(2)]
    try:
        for e in engs:
            e.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
        for e in engs:
            e.update_nodes_delta(np.array([5, 600], dtype=np.int32), np.array([0, 11], dtype=np.int32))
        topo.free[[5, 600]] = [0, 11]
        for e in engs:
            assert repairs(e) == 0
            check_snapshot(e, topo, world1=False)
    finally:
        for e in engs:
            e.close()


def test_delta_behind_an_in_flight_batch():
    """stage + run_staged, then a delta that empties the nodes that batch places on, then fetch: the batch saw the old
    snapshot; the next one sees the new."""
    topo = tg.copy_topo(tg.make("hubs").topo)
    eng = new_engine(topo)
    try:
        blob = _steps(topo, 11, 8)
        old = oracle_placer.place(topo, blob, want_matrix=False, want_topk=False)
        picked = np.unique(old["assign"][old["assign"] >= 0])
        assert len(picked) > 0
        h = eng.stage(blob)
        eng.run_staged(h, 1)
        eng.update_nodes_delta(picked.astype(np.int32), np.zeros(len(picked), dtype=np.int32))
        a, s, d = eng.fetch(h)
        assert np.array_equal(a, old["assign"]) and np.array_equal(s, old["status"]) and np.array_equal(d, old["domain"])
        eng.release(h)
        topo.free[picked] = 0
        check_snapshot(eng, topo)
        new = check_batch(eng, topo, blob, check_matrix=False)
        assert not np.array_equal(new["assign"], old["assign"])
    finally:
        eng.close()


# ---------------------------------------------------------------- library switches
@pytest.mark.parametrize("var", ["RBGTOPO_WIDE_SORT_KEY", "RBGTOPO_SMALL_SORT", "RBGTOPO_NO_REFRESH_GRAPH", "RBGTOPO_NO_DELTA"])
def test_snapshot_variants_in_a_subprocess(var):
    """The library reads its switches when it loads, hence the subprocess.  RBGTOPO_WIDE_SORT_KEY: the plain 64-bit key
    instead of the compact one.  RBGTOPO_SMALL_SORT: slabs of <= 16 384 nodes sorted by one CTA (k_order_sort_small).
    RBGTOPO_NO_REFRESH_GRAPH: plain launches instead of the captured refresh graph.  RBGTOPO_NO_DELTA: every
    update_nodes_delta refreshes fully (the tests then expect no repair).  Runs this file and tests/test_gpu_delta.py."""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ)
    env[var] = "1"
    r = subprocess.run([sys.executable, "-m", "pytest", "tests/test_gpu_snapshot.py", "tests/test_gpu_delta.py", "-q", "-m", "gpu",
                        "-x", "-k", "not subprocess"], cwd=root, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert "passed" in r.stdout
