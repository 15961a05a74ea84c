"""CPU: the plugin mirror's exclusive_keys (DESIGN.md §3.9): groups are hinted only at the level-0 key; any other key
gets no hint and a logged reason, None keeps the behaviour without levels."""
import numpy as np

from rbg_b200 import synth
from rbg_b200.ingest import DEFAULT_TIER_LABELS
from rbg_b200.plugin import (EXCLUSIVE_TOPOLOGY_KEY, RBGTOPO_NO_HINT, B200TopoPodGroupManager, RoleBasedGroup,
                             RoleSpec)
from test_plugin_host import OraclePlacer

NV = DEFAULT_TIER_LABELS[0]
HOSTNAME, ZONE = "kubernetes.io/hostname", "topology.kubernetes.io/zone"


def rbg(name, gid, key=None):
    ann = {EXCLUSIVE_TOPOLOGY_KEY: key} if key is not None else {}
    return RoleBasedGroup("ns", name, [RoleSpec("prefill", 2, (), 1), RoleSpec("decode", 1, ("prefill",), 1)],
                          annotations=ann, gid=gid)


def test_only_the_level0_key_gets_a_hint():
    topo = synth.make_topology(256, seed=5, tiers=3)
    groups = [rbg("a", 1, NV), rbg("b", 2, HOSTNAME), rbg("c", 3, "example.com/rack"), rbg("d", 4)]
    pl = OraclePlacer(topo)
    mgr = B200TopoPodGroupManager(pl, exclusive_keys=[NV, HOSTNAME, ZONE])
    out = mgr.reconcile_pod_groups_by_waves(groups)
    assert [p.status for p in out][1:3] == [RBGTOPO_NO_HINT, RBGTOPO_NO_HINT]
    assert out[0].status == 0 and out[3].status == 0 and all(v >= 0 for v in out[0].nodes.values())
    assert "not the level-0 label" in mgr.no_hint[("ns", "b")] and "not configured" in mgr.no_hint[("ns", "c")]
    # only the hinted groups were marshalled, and only they get the hint annotation
    assert sorted({int(x) for b in pl.blobs for x in b[8:8 + 16 * int(b[2]):16]}) == [1, 4]
    for g, hinted in zip(groups, (True, False, False, True)):
        tmpl = {}
        mgr.InjectPodGroupLabels(g, tmpl)
        assert ("annotations" in tmpl.get("metadata", {})) == hinted, g.name


def test_none_keeps_every_key_at_level0():
    topo = synth.make_topology(256, seed=5, tiers=3)
    groups = [rbg("a", 1, NV), rbg("b", 2, HOSTNAME)]
    out_none = B200TopoPodGroupManager(OraclePlacer(topo)).reconcile_pod_groups_by_waves(groups)
    assert all(p.status == 0 for p in out_none)
    out_same = B200TopoPodGroupManager(OraclePlacer(topo), exclusive_keys=[NV, HOSTNAME]).reconcile_pod_groups_by_waves(groups[:1])
    assert out_same[0] == out_none[0]
