"""CPU: the plugin mirror places exclusive groups at the level their key names when the placer does (DESIGN.md §3.9):
the blob carries the key's index at GROUPS word +10 and step word +14, committed batches still withhold those hints,
and a placer without `places_levels` behaves as before."""
import numpy as np

from rbg_b200 import synth
from rbg_b200.ingest import DEFAULT_TIER_LABELS
from rbg_b200.plugin import (EXCLUSIVE_TOPOLOGY_KEY, RBGTOPO_NO_HINT, B200TopoPodGroupManager, RoleBasedGroup,
                             RoleSpec)
from test_plugin_host import OraclePlacer

NV = DEFAULT_TIER_LABELS[0]
HOSTNAME, ZONE = "kubernetes.io/hostname", "topology.kubernetes.io/zone"
KEYS = [NV, HOSTNAME, ZONE]


class LevelsPlacer:
    """Records the blobs it is given and answers every replica unplaced: what the plugin marshals is under test."""
    places_levels = True

    def __init__(self, n_nodes=256):
        self.n_nodes = n_nodes
        self.blobs = []

    def score_assign(self, blob):
        self.blobs.append(np.array(blob))
        ns = int(blob[2])
        return np.full(int(blob[4]), -1, np.int32), np.ones(ns, np.int32), np.full(ns, -1, np.int32)

    def place_groups(self, gb):
        self.blobs.append(np.array(gb))
        ng = int(gb[2])
        return np.full(int(gb[4]), -1, np.int32), np.ones(ng, np.int32), np.full(ng, -1, np.int32)

    def place_groups_committed(self, gb):
        a, s, d = self.place_groups(gb)
        return a, s, d, 1


def rbg(name, gid, key=None):
    ann = {EXCLUSIVE_TOPOLOGY_KEY: key} if key is not None else {}
    return RoleBasedGroup("ns", name, [RoleSpec("prefill", 2, (), 1), RoleSpec("decode", 1, ("prefill",), 1)],
                          annotations=ann, gid=gid)


def groups():
    return [rbg("a", 1, NV), rbg("b", 2, HOSTNAME), rbg("c", 3, ZONE), rbg("d", 4), rbg("e", 5, "example.com/rack")]


def test_groups_blob_carries_the_key_index():
    pl = LevelsPlacer()
    mgr = B200TopoPodGroupManager(pl, exclusive_keys=KEYS)
    out = mgr.reconcile_pod_groups(groups())
    assert [p.status for p in out] == [1, 1, 1, 1, RBGTOPO_NO_HINT]
    gb = pl.blobs[-1]
    recs = [gb[8 + 12 * g: 8 + 12 * g + 12] for g in range(int(gb[2]))]
    assert [(int(r[0]), int(r[10])) for r in recs] == [(1, 0), (2, 1), (3, 2), (4, 0)]
    assert set(mgr.no_hint) == {("ns", "e")}


def test_steps_carry_the_key_index():
    pl = LevelsPlacer()
    mgr = B200TopoPodGroupManager(pl, exclusive_keys=KEYS)
    out = mgr.reconcile_pod_groups_by_waves(groups())
    assert [p.status for p in out][:4] != [RBGTOPO_NO_HINT] * 4 and out[4].status == RBGTOPO_NO_HINT
    levels = {}
    for b in pl.blobs:
        for s in range(int(b[2])):
            st = b[8 + 16 * s: 8 + 16 * s + 16]
            levels.setdefault(int(st[0]), set()).add(int(st[14]))
    assert levels == {1: {0}, 2: {1}, 3: {2}, 4: {0}}


def test_committed_batches_withhold_level_hints():
    pl = LevelsPlacer()
    mgr = B200TopoPodGroupManager(pl, exclusive_keys=KEYS)
    out = mgr.reconcile_pod_groups(groups(), committed=True)
    assert [p.status for p in out] == [1, RBGTOPO_NO_HINT, RBGTOPO_NO_HINT, 1, RBGTOPO_NO_HINT]
    assert "committed" in mgr.no_hint[("ns", "b")] and "committed" in mgr.no_hint[("ns", "c")]
    gb = pl.blobs[-1]
    assert [int(gb[8 + 12 * g]) for g in range(int(gb[2]))] == [1, 4]


def test_placer_without_the_attribute_keeps_the_level0_path():
    topo = synth.make_topology(256, seed=5, tiers=3)
    pl = OraclePlacer(topo)
    assert not hasattr(pl, "places_levels")
    mgr = B200TopoPodGroupManager(pl, exclusive_keys=KEYS)
    out = mgr.reconcile_pod_groups_by_waves(groups())
    assert [p.status for p in out][1:3] == [RBGTOPO_NO_HINT, RBGTOPO_NO_HINT]
    assert "no placement at that level yet" in mgr.no_hint[("ns", "b")]
    assert all(int(b[8 + 16 * s + 14]) == 0 for b in pl.blobs for s in range(int(b[2])))
