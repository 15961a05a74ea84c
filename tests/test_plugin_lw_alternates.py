"""CPU: the plugin mirror's alternates for leader-worker groups (DESIGN.md §3.12).  With alternates > 0 and a placer
that has `places_lw_ranked`, a group with a multi-pod role is placed through place_groups_lw_ranked: the alternates
annotation is keyed by pod name ("{rbg}-{role}-{ordinal}-{k}"), standalone roles keep the RoleID, and a failed gang
carries none.  A placer without the attribute keeps the no-hint reason."""
import json

import numpy as np

import lw_alternates_oracle as lwa
from alternates_oracle import run_fleet_ranked
from oracle import wave_loop
from rbg_b200.plugin import (GANG_SCHEDULING_KEY, PLACEMENT_ALTERNATES_KEY, RBGTOPO_NO_HINT, B200TopoPodGroupManager,
                             RoleBasedGroup, RoleSpec)
from test_plugin_lw import HOSTNAME, NV, RACK, LwPlacer, lws_group, plain_group, topo_and_levels


class LwRankedPlacer(LwPlacer):
    """LwPlacer plus the ranked calls, answered by the CPU oracles of §3.10 and §3.12."""
    places_lw_ranked = True

    def __init__(self, topo, level_domain=None):
        super().__init__(topo, level_domain)
        self.ranked_calls = []

    def place_groups_ranked(self, gb, n_alt):
        self.ranked_calls.append("place_groups_ranked")
        return run_fleet_ranked(self.topo, wave_loop.groups_from_blob(gb), n_alt)

    def place_groups_lw_ranked(self, gb, role_pods, n_alt):
        self.ranked_calls.append("place_groups_lw_ranked")
        self.lw_calls.append(np.asarray(role_pods).reshape(-1, 2))
        return lwa.run_lw_ranked(self.topo, gb, role_pods, n_alt, level_domain=self.level_domain)


def _annotation(mgr, rbg):
    tmpl = {}
    mgr.InjectPodGroupLabels(rbg, tmpl)
    return json.loads(tmpl["metadata"]["annotations"].get(PLACEMENT_ALTERNATES_KEY, "{}"))


def test_alternates_keyed_by_pod_name_inside_the_colocation_domain():
    topo, lv = topo_and_levels()
    topo.free[:] = 2
    pl = LwRankedPlacer(topo, lv)
    mgr = B200TopoPodGroupManager(pl, exclusive_keys=[NV, HOSTNAME, RACK], alternates=3, leader_worker=True)
    a, b = lws_group("a", 1, RACK, lws=4), plain_group("b", 2)
    out = mgr.reconcile_pod_groups([a, b])
    assert pl.ranked_calls == ["place_groups_ranked", "place_groups_lw_ranked"]
    assert out[0].status != RBGTOPO_NO_HINT and ("ns", "a") not in mgr.no_hint
    alts = _annotation(mgr, a)
    pods = {f"a-decode-{o}-{k}" for o in range(2) for k in range(4)}
    assert set(out[0].nodes) == pods | {"a-router-0"}
    assert set(alts) <= set(out[0].nodes) and set(alts) & pods and "a-router-0" in alts
    for key, nodes in alts.items():
        assert 1 <= len(nodes) <= 3 and out[0].nodes[key] not in nodes
        if key in pods:   # inside the replica's rack
            assert {int(lv[2][m]) for m in nodes} == {int(lv[2][out[0].nodes[key]])}
    assert set(_annotation(mgr, b)) <= {"b-prefill-0", "b-prefill-1", "b-decode-0"} and _annotation(mgr, b)


def test_failed_gang_has_no_alternates():
    topo, _ = topo_and_levels(8)
    topo.free[:] = 1
    pl = LwRankedPlacer(topo)
    mgr = B200TopoPodGroupManager(pl, alternates=2, leader_worker=True)
    gang = RoleBasedGroup("ns", "g", [RoleSpec("decode", 3, (), 1, lws_size=4)],
                          annotations={GANG_SCHEDULING_KEY: "true"}, gid=1)
    ok = lws_group("ok", 2)
    out = mgr.reconcile_pod_groups([gang, ok])
    assert pl.ranked_calls == ["place_groups_lw_ranked"]
    assert out[0].status == 2 and not out[0].alternates.get("g-decode-0-0") and not _annotation(mgr, gang)
    assert _annotation(mgr, ok)


def test_placer_without_ranked_leader_worker_keeps_the_reason():
    topo, _ = topo_and_levels()
    pl = LwPlacer(topo)
    mgr = B200TopoPodGroupManager(pl, alternates=2, leader_worker=True)
    out = mgr.reconcile_pod_groups([lws_group("y", 6)])
    assert out[0].status == RBGTOPO_NO_HINT and "alternates" in mgr.no_hint[("ns", "y")]
    assert not pl.lw_calls
    # committed batches keep their reason with a ranked placer too
    ranked = B200TopoPodGroupManager(LwRankedPlacer(topo), alternates=2, leader_worker=True)
    out = ranked.reconcile_pod_groups([lws_group("x", 5)], committed=True)
    assert out[0].status == RBGTOPO_NO_HINT and "committed" in ranked.no_hint[("ns", "x")]
