"""CPU: committed batches with leader-worker groups in the plugin mirror (DESIGN.md §3.13).  On a placer with
`places_lw_committed`, a committed batch with a multi-pod group and no group at an exclusive level >= 1 goes through one
place_groups_lw_committed call in the given order — standalone groups with (1, -1) for every role and RoleID keys,
leader-worker groups keyed by pod name — and its hints never over-commit a node.  Levels >= 1 and placers without
the attribute keep their no-hint reasons."""
import numpy as np

from lw_committed_oracle import run_lw_committed
from rbg_b200.blob import STEP_EXCLUSIVE
from rbg_b200.plugin import EXCLUSIVE_TOPOLOGY_KEY, RBGTOPO_NO_HINT, B200TopoPodGroupManager
from test_plugin_lw import HOSTNAME, NV, RACK, LwPlacer, lws_group, plain_group, topo_and_levels


class LwCommitPlacer(LwPlacer):
    """LwPlacer plus place_groups_lw_committed answered by the CPU oracle of §3.13; records every call."""
    places_lw_committed = True

    def __init__(self, topo, level_domain=None):
        super().__init__(topo, level_domain)
        self.commit_calls = []

    def place_groups_lw_committed(self, gb, role_pods):
        rp = np.asarray(role_pods).reshape(-1, 2)
        self.commit_calls.append((np.asarray(gb), rp))
        return (*run_lw_committed(self.topo, gb, rp, level_domain=self.level_domain), 1)


def demand_per_node(topo, out, groups):
    used = np.zeros(topo.n, dtype=np.int64)
    for p, g in zip(out, groups):
        demand = {r.name: r.demand for r in g.roles}
        for key, node in p.nodes.items():
            if node >= 0:
                used[node] += demand[key.split("-")[1]]
    return used


def test_a_mixed_batch_is_one_call_in_order():
    topo, lv = topo_and_levels()
    pl = LwCommitPlacer(topo, lv)
    mgr = B200TopoPodGroupManager(pl, exclusive_keys=[NV, HOSTNAME, RACK], leader_worker=True)
    groups = [plain_group("b", 2), lws_group("a", 1, RACK, lws=4), plain_group("d", 4), lws_group("c", 3)]
    out = mgr.reconcile_pod_groups(groups, committed=True)
    assert len(pl.commit_calls) == 1 and not pl.lw_calls and pl.plain_calls == 0
    gb, rp = pl.commit_calls[0]
    assert [int(gb[8 + 12 * g]) for g in range(int(gb[2]))] == [2, 1, 4, 3]
    # roles in (level, name) order: plain (prefill, decode), lws (decode, router)
    assert rp.tolist() == [[1, -1], [1, -1], [4, 2], [1, -1], [1, -1], [1, -1], [2, -1], [1, -1]]
    b, a, d, c = out
    assert set(b.nodes) == {"b-prefill-0", "b-prefill-1", "b-decode-0"}
    assert set(a.nodes) == {f"a-decode-{o}-{k}" for o in range(2) for k in range(4)} | {"a-router-0"}
    assert set(d.nodes) == {"d-prefill-0", "d-prefill-1", "d-decode-0"}
    assert set(c.nodes) == {f"c-decode-{o}-{k}" for o in range(2) for k in range(2)} | {"c-router-0"}


def test_the_hints_of_a_batch_never_over_commit_a_node():
    topo, lv = topo_and_levels(32)
    topo.free[:] = 1
    pl = LwCommitPlacer(topo, lv)
    mgr = B200TopoPodGroupManager(pl, exclusive_keys=[NV, HOSTNAME, RACK], leader_worker=True)
    groups = [lws_group(f"g{i}", i, RACK if i % 2 else None, lws=4) if i % 3 else plain_group(f"g{i}", i)
              for i in range(8)]
    out = mgr.reconcile_pod_groups(groups, committed=True)
    used = demand_per_node(topo, out, groups)
    assert (used <= topo.free).all() and used.sum() > 0
    # the same groups under snapshot semantics collide
    snap = mgr.reconcile_pod_groups(groups)
    assert (demand_per_node(topo, snap, groups) > topo.free).any()


def test_levels_and_placers_without_the_attribute_keep_their_reasons():
    topo, lv = topo_and_levels()
    racked = plain_group("r", 9)
    racked.annotations[EXCLUSIVE_TOPOLOGY_KEY] = RACK
    pl = LwCommitPlacer(topo, lv)
    pl.places_levels = pl.places_committed_levels = True
    mgr = B200TopoPodGroupManager(pl, exclusive_keys=[NV, HOSTNAME, RACK], leader_worker=True)
    out = mgr.reconcile_pod_groups([lws_group("x", 5), racked], committed=True)
    assert not pl.commit_calls
    assert out[0].status == RBGTOPO_NO_HINT and "committed" in mgr.no_hint[("ns", "x")]
    old = LwPlacer(topo, lv)
    mgr = B200TopoPodGroupManager(old, leader_worker=True)
    out = mgr.reconcile_pod_groups([lws_group("y", 6), plain_group("p", 4)], committed=True)
    assert out[0].status == RBGTOPO_NO_HINT and "committed" in mgr.no_hint[("ns", "y")]
    assert out[1].status != RBGTOPO_NO_HINT


def test_exclusive_groups_keep_their_domains_apart():
    topo, lv = topo_and_levels()
    pl = LwCommitPlacer(topo, lv)
    mgr = B200TopoPodGroupManager(pl, leader_worker=True)
    groups = [lws_group(f"e{i}", 10 + i, lws=2, ann={EXCLUSIVE_TOPOLOGY_KEY: NV}) for i in range(4)]
    out = mgr.reconcile_pod_groups(groups, committed=True)
    gb, _ = pl.commit_calls[0]
    assert all(int(gb[8 + 12 * g + 1]) & STEP_EXCLUSIVE for g in range(4))
    doms = [p.domain for p in out if p.domain >= 0]
    assert len(doms) == len(set(doms)) > 1
