"""CPU: committed batches with leader-worker groups and groups at exclusive levels >= 1 in the plugin mirror
(DESIGN.md §3.16).  On a placer with `places_lw_committed_levels` such a batch is one place_groups_lw_committed call
with every group at the level its key names; a placer without the attribute keeps every current reason."""
import numpy as np

import levels_oracle as lo
from lw_committed_levels_oracle import run_lw_committed_levels
from rbg_b200.plugin import EXCLUSIVE_TOPOLOGY_KEY, RBGTOPO_NO_HINT, B200TopoPodGroupManager
from test_plugin_lw import HOSTNAME, NV, RACK, lws_group, plain_group, topo_and_levels
from test_plugin_lw_committed import LwCommitPlacer


class LwCommitLevelsPlacer(LwCommitPlacer):
    """place_groups_lw_committed answered by the CPU oracle of §3.16 (no occupancy records)."""
    places_levels = places_committed_levels = places_lw_committed_levels = True

    def place_groups_lw_committed(self, gb, role_pods):
        rp = np.asarray(role_pods).reshape(-1, 2)
        self.commit_calls.append((np.asarray(gb), rp))
        lv = np.asarray(self.level_domain)
        nd = [int(x.max()) + 1 for x in lv]
        owner = lo.derive_level_owner(lv, np.zeros((0, 3), np.int32))
        return (*run_lw_committed_levels(self.topo, gb, rp, lv, owner, nd), 1)


def racked(name, gid):
    g = plain_group(name, gid)
    g.annotations[EXCLUSIVE_TOPOLOGY_KEY] = RACK
    return g


def test_a_batch_with_a_rack_keyed_group_is_one_call():
    topo, lv = topo_and_levels()
    pl = LwCommitLevelsPlacer(topo, lv)
    mgr = B200TopoPodGroupManager(pl, exclusive_keys=[NV, HOSTNAME, RACK], leader_worker=True)
    out = mgr.reconcile_pod_groups([lws_group("x", 5), racked("r", 9), lws_group("y", 6, RACK, lws=4)],
                                   committed=True)
    assert len(pl.commit_calls) == 1 and not mgr.no_hint
    gb, rp = pl.commit_calls[0]
    assert [int(gb[8 + 12 * g + 10]) for g in range(int(gb[2]))] == [0, 2, 0]
    assert all(p.status != RBGTOPO_NO_HINT for p in out)
    assert set(out[0].nodes) == {f"x-decode-{o}-{k}" for o in range(2) for k in range(2)} | {"x-router-0"}
    assert set(out[1].nodes) == {"r-prefill-0", "r-prefill-1", "r-decode-0"}


def test_placers_without_the_attribute_keep_their_reasons():
    topo, lv = topo_and_levels()
    pl = LwCommitPlacer(topo, lv)
    pl.places_levels = pl.places_committed_levels = True
    mgr = B200TopoPodGroupManager(pl, exclusive_keys=[NV, HOSTNAME, RACK], leader_worker=True)
    out = mgr.reconcile_pod_groups([lws_group("x", 5), racked("r", 9)], committed=True)
    assert not pl.commit_calls
    assert out[0].status == RBGTOPO_NO_HINT and "committed" in mgr.no_hint[("ns", "x")]
    pl = LwCommitLevelsPlacer(topo, lv)
    pl.places_committed_levels = False       # the rack-keyed group itself still needs committed levels
    mgr = B200TopoPodGroupManager(pl, exclusive_keys=[NV, HOSTNAME, RACK], leader_worker=True)
    out = mgr.reconcile_pod_groups([lws_group("x", 5), racked("r", 9)], committed=True)
    assert out[1].status == RBGTOPO_NO_HINT and "level 0 only" in mgr.no_hint[("ns", "r")]
    assert out[0].status != RBGTOPO_NO_HINT
