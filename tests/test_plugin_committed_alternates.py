"""CPU: the plugin mirror's alternates for committed batches (DESIGN.md §3.14).  With alternates > 0 and a placer that
has `places_committed_ranked`, reconcile_pod_groups(committed=True) goes through place_groups_committed_ranked and the
alternates annotation is present, keyed by RoleID; the hints are those of place_groups_committed.  A placer without
the attribute keeps the committed hints byte for byte, without alternates."""
import json

import numpy as np

import committed_alternates_oracle as cao
from committed_oracle import result_arrays, run_fleet_committed
from oracle import wave_loop
from rbg_b200 import synth
from rbg_b200.plugin import PLACEMENT_ALTERNATES_KEY, RBGTOPO_NO_HINT, B200TopoPodGroupManager
from test_plugin_host import OraclePlacer
from test_plugin_lw import plain_group


class CommittedPlacer(OraclePlacer):
    """place_groups_committed answered by the committed oracle (§3.8)."""

    def __init__(self, topo):
        super().__init__(topo)
        self.calls = []

    def place_groups_committed(self, gb):
        self.calls.append("place_groups_committed")
        a, s, d = result_arrays(run_fleet_committed(self.topo, wave_loop.groups_from_blob(gb)))
        return a, s, d, 1


class CommittedRankedPlacer(CommittedPlacer):
    places_committed_ranked = True

    def place_groups_committed_ranked(self, gb, n_alt):
        self.calls.append("place_groups_committed_ranked")
        a, s, d, score, alt, alt_s = cao.run_fleet_committed_ranked(self.topo, wave_loop.groups_from_blob(gb), n_alt)
        return a, s, d, 1, score, alt, alt_s


def _topo():
    topo = synth.make_topology(48, seed=6, tiers=2, max_free=2)
    topo.domain_owner[:] = -1
    return topo


def _annotations(mgr, rbg):
    tmpl = {}
    mgr.InjectPodGroupLabels(rbg, tmpl)
    return tmpl["metadata"]["annotations"]


def test_committed_batch_with_alternates_keyed_by_role_id():
    topo = _topo()
    groups = [plain_group(f"g{i}", i) for i in range(4)]
    pl = CommittedRankedPlacer(topo)
    mgr = B200TopoPodGroupManager(pl, alternates=3)
    out = mgr.reconcile_pod_groups(groups, committed=True)
    assert pl.calls == ["place_groups_committed_ranked"]
    ref = B200TopoPodGroupManager(CommittedPlacer(topo)).reconcile_pod_groups(groups, committed=True)
    used = np.zeros(topo.n, np.int64)
    for p in out:
        for node in p.nodes.values():
            if node >= 0:
                used[node] += 1
    for g, p, r in zip(groups, out, ref):
        assert p.status != RBGTOPO_NO_HINT and p.nodes == r.nodes and p.status == r.status
        alts = json.loads(_annotations(mgr, g)[PLACEMENT_ALTERNATES_KEY])
        assert set(alts) <= set(p.nodes) and alts
        for key, nodes in alts.items():
            assert len(nodes) <= 3 and p.nodes[key] not in nodes
            assert all(used[m] + 1 <= topo.free[m] for m in nodes)   # room once the whole batch is placed


def test_placer_without_the_capability_keeps_todays_hints():
    topo = _topo()
    groups = [plain_group(f"g{i}", i) for i in range(4)]
    plain = CommittedPlacer(topo)
    mgr = B200TopoPodGroupManager(plain, alternates=3)
    out = mgr.reconcile_pod_groups(groups, committed=True)
    assert plain.calls == ["place_groups_committed"]
    base = B200TopoPodGroupManager(CommittedPlacer(topo), alternates=0)
    ref = base.reconcile_pod_groups(groups, committed=True)
    for g, p, r in zip(groups, out, ref):
        assert p == r
        assert _annotations(mgr, g) == _annotations(base, g)
        assert PLACEMENT_ALTERNATES_KEY not in _annotations(mgr, g)
