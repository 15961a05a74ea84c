"""CPU: alternates for committed batches with leader-worker groups in the plugin mirror (DESIGN.md §3.15).  With
alternates > 0 and a placer that has `places_lw_committed_ranked`, a committed batch that takes the leader-worker route
goes through one place_groups_lw_committed_ranked call: its hints are place_groups_lw_committed's, and every group of
the batch carries alternates — one-pod groups keyed by RoleID, multi-pod groups by pod name.  A placer without the
attribute gives exactly the hints it gave before, without alternates."""
import json

import numpy as np

from lw_committed_alternates_oracle import run_lw_committed_ranked
from rbg_b200.plugin import PLACEMENT_ALTERNATES_KEY, RBGTOPO_NO_HINT, B200TopoPodGroupManager
from test_plugin_lw import HOSTNAME, NV, RACK, lws_group, plain_group, topo_and_levels
from test_plugin_lw_committed import LwCommitPlacer, demand_per_node


class LwCommitRankedPlacer(LwCommitPlacer):
    """LwCommitPlacer plus place_groups_lw_committed_ranked answered by the CPU oracle of §3.15."""
    places_lw_ranked = True
    places_lw_committed_ranked = True

    def __init__(self, topo, level_domain=None):
        super().__init__(topo, level_domain)
        self.ranked_calls = []

    def place_groups_lw_committed_ranked(self, gb, role_pods, n_alt):
        rp = np.asarray(role_pods).reshape(-1, 2)
        self.ranked_calls.append((np.asarray(gb), rp, n_alt))
        a, s, d, score, alt, alt_s = run_lw_committed_ranked(self.topo, gb, rp, n_alt, level_domain=self.level_domain)
        return a, s, d, 1, score, alt, alt_s


class LwCommitOnlyPlacer(LwCommitPlacer):
    """A placer from before the ranked committed leader-worker call: it ranks leader-worker groups on their own."""
    places_lw_ranked = True


def _annotations(mgr, rbg):
    tmpl = {}
    mgr.InjectPodGroupLabels(rbg, tmpl)
    return tmpl["metadata"]["annotations"]


def _batch():
    return [plain_group("b", 2), lws_group("a", 1, RACK, lws=4), plain_group("d", 4), lws_group("c", 3)]


def test_a_mixed_batch_gets_alternates_for_every_group():
    topo, lv = topo_and_levels()
    pl = LwCommitRankedPlacer(topo, lv)
    mgr = B200TopoPodGroupManager(pl, exclusive_keys=[NV, HOSTNAME, RACK], leader_worker=True, alternates=3)
    groups = _batch()
    out = mgr.reconcile_pod_groups(groups, committed=True)
    assert len(pl.ranked_calls) == 1 and not pl.commit_calls and not pl.lw_calls and pl.plain_calls == 0
    gb, rp, n_alt = pl.ranked_calls[0]
    assert n_alt == 3 and [int(gb[8 + 12 * g]) for g in range(int(gb[2]))] == [2, 1, 4, 3]
    ref = B200TopoPodGroupManager(LwCommitPlacer(topo, lv), exclusive_keys=[NV, HOSTNAME, RACK],
                                  leader_worker=True).reconcile_pod_groups(groups, committed=True)
    used = demand_per_node(topo, out, groups)
    for g, p, r in zip(groups, out, ref):
        assert p.status != RBGTOPO_NO_HINT and p.nodes == r.nodes and p.status == r.status and p.domain == r.domain
        alts = json.loads(_annotations(mgr, g)[PLACEMENT_ALTERNATES_KEY])
        assert alts and set(alts) <= set(p.nodes)
        for key, nodes in alts.items():
            assert len(nodes) <= 3 and p.nodes[key] not in nodes
            assert all(used[m] + 1 <= topo.free[m] for m in nodes)   # room once the whole batch is placed
    b, a, d, c = (set(json.loads(_annotations(mgr, g)[PLACEMENT_ALTERNATES_KEY])) for g in groups)
    assert b <= {"b-prefill-0", "b-prefill-1", "b-decode-0"} and d <= {"d-prefill-0", "d-prefill-1", "d-decode-0"}
    assert any(k.count("-") == 3 for k in a) and any(k.count("-") == 3 for k in c)   # "{rbg}-{role}-{ordinal}-{k}"
    for key, nodes in json.loads(_annotations(mgr, groups[1])[PLACEMENT_ALTERNATES_KEY]).items():
        if key.startswith("a-decode-"):                                            # co-located in a rack
            assert all(lv[2][m] == lv[2][out[1].nodes[key]] for m in nodes)


def test_a_placer_without_the_attribute_gives_todays_hints():
    topo, lv = topo_and_levels()
    groups = _batch()
    old = LwCommitOnlyPlacer(topo, lv)
    mgr = B200TopoPodGroupManager(old, exclusive_keys=[NV, HOSTNAME, RACK], leader_worker=True, alternates=3)
    out = mgr.reconcile_pod_groups(groups, committed=True)
    assert len(old.commit_calls) == 1
    base = B200TopoPodGroupManager(LwCommitOnlyPlacer(topo, lv), exclusive_keys=[NV, HOSTNAME, RACK],
                                   leader_worker=True)
    ref = base.reconcile_pod_groups(groups, committed=True)
    for g, p, r in zip(groups, out, ref):
        assert p == r
        assert _annotations(mgr, g) == _annotations(base, g)
        assert PLACEMENT_ALTERNATES_KEY not in _annotations(mgr, g)
