"""CPU: the ranked-placement oracle (tests/alternates_oracle.py, DESIGN.md §3.10) — its invariants on generated and
contended fleets, hand-built known answers, and the plugin mirror's `alternates` option over an oracle placer."""
import json

import numpy as np
import pytest

import groups_gen as gg
from alternates_oracle import run_fleet_ranked
from oracle import wave_loop
from rbg_b200 import synth
from rbg_b200.plugin import (PLACEMENT_ALTERNATES_KEY, PLACEMENT_HINT_KEY, B200TopoPodGroupManager,
                             RoleBasedGroup, RoleSpec)


def uniform_topology(n, free, domain):
    """Complete graph with every edge weight 1: equal free capacity gives every node the same score."""
    rp, ci = [0], []
    for v in range(n):
        ci.extend(u for u in range(n) if u != v)
        rp.append(len(ci))
    owner = -np.ones(max(domain) + 1, dtype=np.int32)
    return synth.Topology(np.asarray(rp, np.int32), np.asarray(ci, np.int32), np.ones(len(ci), np.int32),
                          np.asarray(free, np.int32), np.asarray(domain, np.int32), owner)


def check_invariants(topo, groups, n_alt):
    a, s, d, score, alt, alt_s = run_fleet_ranked(topo, groups, n_alt)
    states, _ = wave_loop.run_fleet(topo, groups)
    ref = np.concatenate([st.assign_in_group_order() for st in states]).astype(np.int32)
    assert np.array_equal(a, ref)
    free = np.asarray(topo.free, np.int64)
    off = 0
    for gi, st in enumerate(states):
        used = np.zeros(topo.n, np.int64)
        reps = []
        for ri in st.order:
            for _ in range(st.pending[ri]):
                reps.append((off, st.g.roles[ri]))
                if a[off] >= 0:
                    used[a[off]] += st.g.roles[ri].demand
                off += 1
        for r, role in reps:
            nodes = [int(x) for x in alt[r] if x >= 0]
            k = len(nodes)
            assert list(alt[r][k:]) == [-1] * (n_alt - k) and np.all(alt_s[r][k:] == -np.inf)
            if a[r] < 0:
                assert score[r] == -np.inf and k == 0
                continue
            assert score[r] != -np.inf
            assert len(set(nodes)) == k and a[r] not in nodes
            for n in nodes:
                assert free[n] - used[n] >= role.demand
                if st.g.exclusive and role.exclusive:
                    assert topo.domain[n] == d[gi]
            for i in range(1, k):   # score descending, ties by node ascending
                assert alt_s[r][i] < alt_s[r][i - 1] or (alt_s[r][i] == alt_s[r][i - 1] and nodes[i] > nodes[i - 1])
    return a, s, d, score, alt, alt_s


@pytest.mark.parametrize("seed,n,scarce,excl", [c for c in gg.CASES if c[1] <= 130])
def test_invariants_on_generated_fleets(seed, n, scarce, excl):
    case = gg.make_case(seed, n, scarce=scarce, exclusive=excl)
    for n_alt in (1, 8):
        check_invariants(case.topo, wave_loop.groups_from_blob(case.blob), n_alt)


def test_invariants_on_contended_fleets():
    seen = {"alts": 0, "partial": 0, "gang": 0}
    for seed in range(12):
        rng = np.random.default_rng(seed)
        n = int(rng.integers(6, 40))
        topo = synth.make_topology(n, seed=seed, tiers=2, max_free=3)
        topo.free = np.where(rng.random(n) < 0.6, 0, topo.free).astype(np.int32)   # scarce: partial groups, failed gangs
        groups = [wave_loop.OGroup(f"g{i}", i, [wave_loop.ORole("a", int(rng.integers(1, 9)), demand=1),
                                                wave_loop.ORole("b", int(rng.integers(0, 4)), deps=("a",),
                                                                demand=int(rng.integers(1, 3)),
                                                                exclusive=bool(rng.random() < 0.5))],
                                   exclusive=bool(rng.random() < 0.5), gang=bool(rng.random() < 0.3))
                  for i in range(int(rng.integers(2, 8)))]
        _, s, _, _, alt, _ = check_invariants(topo, groups, 4)
        seen["alts"] += int((alt >= 0).sum())
        seen["partial"] += int((s == 1).sum())
        seen["gang"] += int((s == 2).sum())
    assert all(seen.values()), seen


def test_a_full_neighbour_is_skipped():
    """Two replicas on nodes 0 and 1 of four equal nodes with one slot each: each replica's row is finite on the
    other's node (same wave), but that node has no room once the group is placed."""
    topo = uniform_topology(4, [1, 1, 1, 1], [0, 0, 0, 0])
    g = wave_loop.OGroup("g", 7, [wave_loop.ORole("a", 2, demand=1)])
    a, s, d, score, alt, alt_s = run_fleet_ranked(topo, [g], 3)
    base = 3 * 1 + 8000            # three unit edges to nodes with fmin 1, plus the self term
    assert a.tolist() == [0, 1] and s.tolist() == [0]
    assert score.tolist() == [2 * base, 2 * base]   # need = 2 unplaced replicas of the role
    assert alt.tolist() == [[2, 3, -1], [2, 3, -1]]
    assert alt_s[:, :2].tolist() == [[2 * base] * 2] * 2 and np.all(alt_s[:, 2] == -np.inf)


def test_an_opted_out_role_can_leave_the_domain():
    """Exclusive group: role a (participating) then role b (opted out, depends on a).  Nodes 0, 1 form domain 0 and
    nodes 2, 3 domain 1, two slots each.  a takes node 0 and fixes domain 0; b joins it on node 0, which is then full.
    a's alternates stay in domain 0; b's run across both domains."""
    topo = uniform_topology(4, [2, 2, 2, 2], [0, 0, 1, 1])
    g = wave_loop.OGroup("g", 3, [wave_loop.ORole("a", 1, demand=1, exclusive=True),
                                  wave_loop.ORole("b", 1, deps=("a",), demand=1, exclusive=False)], exclusive=True)
    a, s, d, score, alt, alt_s = run_fleet_ranked(topo, [g], 3)
    assert a.tolist() == [0, 0] and d.tolist() == [0]
    assert alt.tolist() == [[1, -1, -1], [1, 2, 3]]
    assert alt_s[1, 0] == alt_s[1, 1] == alt_s[1, 2] and alt_s[1, 0] < score[1]


class OraclePlacer:
    """place_groups / place_groups_ranked on the oracle (snapshot semantics), with a log of the calls made."""

    def __init__(self, topo):
        self.topo, self.n_nodes, self.calls = topo, topo.n, []

    def place_groups(self, blob):
        self.calls.append("place_groups")
        a, s, d, *_ = run_fleet_ranked(self.topo, wave_loop.groups_from_blob(blob), 0)
        return a, s, d

    def place_groups_ranked(self, blob, n_alt):
        self.calls.append("place_groups_ranked")
        return run_fleet_ranked(self.topo, wave_loop.groups_from_blob(blob), n_alt)


def _rbgs():
    return [RoleBasedGroup("default", f"svc{i}", [RoleSpec("prefill", 2, (), 1), RoleSpec("decode", 3, ("prefill",), 1)],
                           gid=i) for i in range(3)]


def test_plugin_alternates_annotation():
    topo = synth.make_topology(64, seed=4, tiers=2, max_free=2)
    plain_pl, ranked_pl = OraclePlacer(topo), OraclePlacer(topo)
    plain = B200TopoPodGroupManager(plain_pl)
    ranked = B200TopoPodGroupManager(ranked_pl, alternates=3)
    out0, out3 = plain.reconcile_pod_groups(_rbgs()), ranked.reconcile_pod_groups(_rbgs())
    assert plain_pl.calls == ["place_groups"] and ranked_pl.calls == ["place_groups_ranked"]
    assert all(p.alternates == {} for p in out0)
    assert [(p.status, p.nodes, p.domain, p.scores) for p in out0] == [(p.status, p.nodes, p.domain, p.scores)
                                                                      for p in out3]
    assert any(p.alternates for p in out3)
    for r, p0, p3 in zip(_rbgs(), out0, out3):
        t0, t3 = {}, {}
        plain.InjectPodGroupLabels(r, t0)
        ranked.InjectPodGroupLabels(r, t3)
        assert PLACEMENT_ALTERNATES_KEY not in t0["metadata"]["annotations"]
        assert t0["metadata"]["annotations"][PLACEMENT_HINT_KEY] == t3["metadata"]["annotations"][PLACEMENT_HINT_KEY]
        alts = json.loads(t3["metadata"]["annotations"][PLACEMENT_ALTERNATES_KEY])
        assert alts == {k: v for k, v in sorted(p3.alternates.items()) if v}
        assert all(1 <= len(v) <= 3 and p3.nodes[k] not in v for k, v in alts.items())


def test_plugin_default_is_unchanged_and_the_option_is_bounded():
    topo = synth.make_topology(64, seed=5, tiers=2)
    assert B200TopoPodGroupManager(OraclePlacer(topo)).alternates == 0
    for bad in (-1, 9):
        with pytest.raises(ValueError):
            B200TopoPodGroupManager(OraclePlacer(topo), alternates=bad)
