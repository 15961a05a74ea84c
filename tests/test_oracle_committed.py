"""CPU: the oracle of the committed batch (tests/committed_oracle.py, DESIGN.md §3.8) keeps the invariants the
section states — no over-committed node, no exclusive domain shared by two gids unless the caller fixed it, gang
all-or-nothing, group 0 and groups that touch nothing an earlier group took placed as under snapshot semantics —
and gives the known answers of hand-built cases; its fast variant equals the literal one, and in occupancy mode
(DESIGN.md §3.9) its placements keep the records' anti-affinity terms."""
import numpy as np
import pytest

import commit_gen as cg
import groups_gen as gg
import levels_oracle as lo
from committed_oracle import result_arrays, run_fleet_committed, run_fleet_snapshot
from oracle import wave_loop
from rbg_b200 import synth


def placed_per_node(states, n):
    used = np.zeros(n, dtype=np.int64)
    for s in states:
        res = s.result()
        for wave in s.waves:
            for ri, ordinal, cnt in wave:
                for c in range(cnt):
                    node = res["nodes"][f"{s.g.name}-{s.g.roles[ri].name}-{ordinal + c}"]
                    if node >= 0:
                        used[node] += s.g.roles[ri].demand
    return used


def check_invariants(topo, groups, states):
    used = placed_per_node(states, topo.n)
    over = np.nonzero(used > topo.free)[0]
    assert len(over) == 0, ("over-committed", over[:8], used[over[:8]], topo.free[over[:8]])
    chosen = {}   # domain -> gid of the first group that reported it
    for g, s in zip(groups, states):
        res = s.result()
        a = s.assign_in_group_order()
        if g.gang:
            assert (res["status"] == 2 and all(x == -1 for x in a)) or (res["status"] == 0 and all(x >= 0 for x in a)), g.name
        if res["status"] == 2:
            assert all(x == -1 for x in a) and res["domain"] == -1
        if g.exclusive and res["status"] != 2 and res["domain"] >= 0:
            d = res["domain"]
            if d in chosen and chosen[d] != g.gid:
                assert g.fixed_domain == d, ("domain shared by two gids", g.name, d, chosen[d], g.gid)
            chosen.setdefault(d, g.gid)


def same_result(a, b):
    ra, rb = a.result(), b.result()
    return a.assign_in_group_order() == b.assign_in_group_order() and (ra["status"], ra["domain"]) == (rb["status"], rb["domain"])


@pytest.mark.parametrize("seed,n,scarce,excl", [c for c in gg.CASES if c[1] <= 2049])
def test_groups_gen_fleets_keep_the_invariants(seed, n, scarce, excl):
    case = gg.make_case(seed, n, n_groups=12, scarce=scarce, exclusive=excl)
    groups = wave_loop.groups_from_blob(case.blob)
    states = run_fleet_committed(case.topo, groups)
    check_invariants(case.topo, groups, states)
    snap = run_fleet_snapshot(case.topo, groups)
    assert same_result(states[0], snap[0])


def contended(seed, n_nodes=24, n_groups=12, scarce=False, exclusive=False, gang=False):
    """Few nodes, many similar groups: every group wants the head of the same background order."""
    rng = np.random.default_rng(seed)
    topo = synth.make_topology(n_nodes, seed=seed, tiers=2, max_free=3)
    if scarce:
        topo.free = np.where(rng.random(n_nodes) < 0.5, 0, topo.free).astype(np.int32)
    groups = []
    for g in range(n_groups):
        roles = [wave_loop.ORole("a", int(rng.integers(1, 4)), demand=int(rng.integers(1, 3))),
                 wave_loop.ORole("b", int(rng.integers(0, 3)), deps=("a",), demand=1)]
        groups.append(wave_loop.OGroup(f"rbg{g}", 10 + g, roles, exclusive=exclusive, gang=gang or bool(rng.random() < 0.3)))
    return topo, groups


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("scarce,exclusive,gang", [(False, False, False), (True, False, True), (False, True, False),
                                                   (True, True, False)])
def test_contended_fleets_keep_the_invariants(seed, scarce, exclusive, gang):
    topo, groups = contended(seed, scarce=scarce, exclusive=exclusive, gang=gang)
    states = run_fleet_committed(topo, groups)
    check_invariants(topo, groups, states)
    assert same_result(states[0], run_fleet_snapshot(topo, groups[:1])[0])


def test_snapshot_semantics_over_commit_what_committed_does_not():
    """The motivation: under snapshot semantics similar groups ask the same nodes for more than they have."""
    topo, groups = contended(0, n_nodes=16, n_groups=10)
    snap = run_fleet_snapshot(topo, groups)
    assert (placed_per_node(snap, topo.n) > topo.free).any()
    assert not (placed_per_node(run_fleet_committed(topo, groups), topo.n) > topo.free).any()


def test_groups_on_disjoint_nodes_match_snapshot_semantics():
    """Exclusive groups with distinct fixed domains (every role exclusive) never see each other's nodes."""
    topo = synth.make_topology(256, seed=3, tiers=2, max_free=4)
    n_dom = len(topo.domain_owner)
    topo.domain_owner[:] = -1
    rng = np.random.default_rng(3)
    doms = rng.permutation(n_dom)[:8]
    groups = [wave_loop.OGroup(f"rbg{i}", 50 + i,
                               [wave_loop.ORole("p", int(rng.integers(1, 4))), wave_loop.ORole("d", int(rng.integers(1, 4)), deps=("p",))],
                               exclusive=True, fixed_domain=int(d)) for i, d in enumerate(doms)]
    committed = run_fleet_committed(topo, groups)
    snap = run_fleet_snapshot(topo, groups)
    assert all(same_result(a, b) for a, b in zip(committed, snap))
    a, st, dm = result_arrays(committed)
    assert (a >= 0).any() and list(dm) == [int(d) for d in doms]


def line_topology():
    """0 -1000- 1 -100- 2 -10- 3, one slot each: base = 9000, 9100, 8110, 8010 (node 1 best, node 0 next)."""
    row_ptr = np.array([0, 1, 3, 5, 6], dtype=np.int32)
    col = np.array([1, 0, 2, 1, 3, 2], dtype=np.int32)
    w = np.array([1000, 1000, 100, 100, 10, 10], dtype=np.int32)
    return synth.Topology(row_ptr, col, w, np.ones(4, dtype=np.int32), np.zeros(4, dtype=np.int32),
                          np.full(1, -1, dtype=np.int32))


def test_second_group_gets_the_next_best_node():
    topo = line_topology()
    groups = [wave_loop.OGroup(f"rbg{i}", i, [wave_loop.ORole("w", 1)]) for i in range(3)]
    snap = run_fleet_snapshot(topo, groups)
    assert [s.assign_in_group_order() for s in snap] == [[1], [1], [1]]
    committed = run_fleet_committed(topo, groups)
    assert [s.assign_in_group_order() for s in committed] == [[1], [0], [2]]


def test_exclusive_domain_taken_by_an_earlier_group():
    """Two exclusive groups with different gids: the second cannot enter the domain the first reported."""
    topo = line_topology()
    topo.domain = np.array([0, 0, 1, 1], dtype=np.int32)
    topo.domain_owner = np.full(2, -1, dtype=np.int32)
    topo.free = np.full(4, 4, dtype=np.int32)
    groups = [wave_loop.OGroup(f"rbg{i}", 7 + i, [wave_loop.ORole("w", 1)], exclusive=True) for i in range(2)]
    committed = run_fleet_committed(topo, groups)
    assert [s.result()["domain"] for s in committed] == [0, 1]
    assert [s.assign_in_group_order() for s in committed] == [[1], [2]]
    same_gid = [wave_loop.OGroup(f"rbg{i}", 7, [wave_loop.ORole("w", 1)], exclusive=True) for i in range(2)]
    assert [s.result()["domain"] for s in run_fleet_committed(topo, same_gid)] == [0, 0]


def _same_states(a, b):
    return len(a) == len(b) and all(same_result(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("scarce,exclusive,gang", [(False, False, False), (True, False, True), (False, True, False),
                                                   (True, True, False)])
def test_fast_committed_oracle_equals_the_literal_one(seed, scarce, exclusive, gang):
    """The committed loop over oracle_placer.place_fast gives the literal oracle's bits on every contended case."""
    topo, groups = contended(seed, scarce=scarce, exclusive=exclusive, gang=gang)
    assert _same_states(run_fleet_committed(topo, groups, fast=True), run_fleet_committed(topo, groups))


def test_fast_committed_oracle_equals_the_literal_one_on_the_bench_fleet():
    """cfg3's fleet (1 024 groups, 10 000 nodes) up to group 160 through both oracles; the whole batch takes the fast
    oracle about 1 s on one CPU thread."""
    import bench
    from rbg_b200.plugin import B200TopoPodGroupManager

    class Shape:
        n_nodes = 10000
    topo = synth.make_topology(10000, seed=0)
    gblob, _ = B200TopoPodGroupManager(Shape()).groups_blob(bench.to_plugin(bench.fleet_spec("mooncake", 1024, 10000, 0)))
    groups = wave_loop.groups_from_blob(gblob)
    assert _same_states(run_fleet_committed(topo, groups, limit=160, fast=True),
                        run_fleet_committed(topo, groups, limit=160))


KEYS = [f"example.com/level-{L}" for L in range(8)]


def check_records(lv, occ, groups, states):
    """Every placement of an exclusive group's participating role keeps the records' anti-affinity terms."""
    for g, s in zip(groups, states):
        if not g.exclusive:
            continue
        res = s.result()["nodes"]
        for ri, r in enumerate(g.roles):
            if not r.exclusive:
                continue
            for c in range(s.pending[ri]):
                node = res[f"{g.name}-{r.name}-{s.first[ri] + c}"]
                assert node < 0 or not lo.violates(lv, KEYS[:len(lv)], occ, g.gid, 0, node), (g.name, r.name, node)


def test_a_claim_never_unblocks_a_node_the_records_block():
    """DESIGN.md §3.9 known answer: node 1 is blocked for gid 7 by gid 9's rack-keyed record; the first gid-7 group
    reports domain 0 (which holds node 1), and the second gid-7 group still cannot use node 1."""
    topo, lv, occ, _, gblob = cg.known_occupancy()
    owner0 = lo.derive_level_owner(lv, occ)[0]
    assert owner0.tolist() == [-1, 9, 9, 9]
    assert lo.violates(lv, KEYS[:2], occ, 7, 0, 1)
    groups = wave_loop.groups_from_blob(gblob)
    states = run_fleet_committed(topo, groups, owner0=owner0)
    assert [s.assign_in_group_order() for s in states] == [[0], [-1]]
    assert [s.result()["domain"] for s in states] == [0, -1]
    check_records(lv, occ, groups, states)
    assert _same_states(states, run_fleet_committed(topo, groups, owner0=owner0, fast=True))


@pytest.mark.parametrize("i", range(len(cg.occupancy_cases())))
def test_generated_occupancy_batches_keep_the_records(i):
    case, lv, occ, owner0 = cg.occupancy_cases()[i]
    groups = wave_loop.groups_from_blob(case.blob)
    states = run_fleet_committed(case.topo, groups, owner0=owner0, fast=True)
    check_invariants(case.topo, groups, states)
    check_records(lv, occ, groups, states)
