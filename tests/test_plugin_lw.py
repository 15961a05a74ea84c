"""CPU: the plugin mirror's leader-worker option (DESIGN.md §3.11).  With leader_worker=True a group with a role of
lws_size > 1 is placed through place_groups_lw and its hints are keyed by pod name; the co-location annotation
resolves against exclusive_keys; unknown keys, missing levels, committed batches and alternates give no hint and a
reason; leader_worker=False leaves everything as it was."""
import numpy as np

import lw_oracle
from rbg_b200 import synth
from rbg_b200.plugin import (COLOCATE_KEY, RBGTOPO_NO_HINT, B200TopoPodGroupManager, RoleBasedGroup, RoleSpec)
from test_plugin_host import OraclePlacer

NV, HOSTNAME, RACK = "nvlink-domain", "kubernetes.io/hostname", "example.com/rack"


class LwPlacer(OraclePlacer):
    """OraclePlacer plus place_groups_lw answered by the CPU oracle of §3.11; records the (S, C) tables."""

    def __init__(self, topo, level_domain=None):
        super().__init__(topo)
        self.level_domain = level_domain
        self._n_levels = 0 if level_domain is None else len(level_domain) - 1
        self.lw_calls = []
        self.plain_calls = 0

    def place_groups(self, gb):   # §3.11 rule 5: one pod per replica and no co-location is place_groups
        self.plain_calls += 1
        return lw_oracle.run_lw(self.topo, gb, lw_oracle.role_pods_for(gb, lambda g, r: (1, -1)))

    def place_groups_committed(self, gb):   # under test here: which groups reach the call
        return (*self.place_groups(gb), 1)

    def place_groups_lw(self, gb, role_pods):
        self.lw_calls.append(np.asarray(role_pods).reshape(-1, 2))
        return lw_oracle.run_lw(self.topo, gb, role_pods, level_domain=self.level_domain)


def lws_group(name, gid, colocate=None, lws=2, ann=None):
    roles = [RoleSpec("decode", 2, (), 1, lws_size=lws, annotations={COLOCATE_KEY: colocate} if colocate else {}),
             RoleSpec("router", 1, (), 1)]
    return RoleBasedGroup("ns", name, roles, annotations=ann or {}, gid=gid)


def plain_group(name, gid):
    return RoleBasedGroup("ns", name, [RoleSpec("prefill", 2, (), 1), RoleSpec("decode", 1, ("prefill",), 1)], gid=gid)


def topo_and_levels(n=64):
    topo = synth.make_topology(n, seed=3, tiers=2, max_free=2)
    topo.domain_owner[:] = -1
    return topo, [topo.domain, np.arange(n, dtype=np.int32), (np.arange(n) // 16).astype(np.int32)]


def test_pod_keyed_hints_and_colocation_level():
    topo, lv = topo_and_levels()
    pl = LwPlacer(topo, lv)
    mgr = B200TopoPodGroupManager(pl, exclusive_keys=[NV, HOSTNAME, RACK], leader_worker=True)
    out = mgr.reconcile_pod_groups([lws_group("a", 1, RACK, lws=4), plain_group("b", 2), lws_group("c", 3)])
    a, b, c = out
    assert set(a.nodes) == {f"a-decode-{o}-{k}" for o in range(2) for k in range(4)} | {"a-router-0"}
    assert set(b.nodes) == {"b-prefill-0", "b-prefill-1", "b-decode-0"}
    assert set(c.nodes) == {f"c-decode-{o}-{k}" for o in range(2) for k in range(2)} | {"c-router-0"}
    # one leader-worker call for a and c (roles in (level, name) order: decode, router), b through place_groups
    assert len(pl.lw_calls) == 1 and pl.plain_calls == 1
    assert pl.lw_calls[0].tolist() == [[4, 2], [1, -1], [2, -1], [1, -1]]
    for o in range(2):   # a replica's pods share one rack, or are all unplaced
        pods = [a.nodes[f"a-decode-{o}-{k}"] for k in range(4)]
        assert all(p >= 0 for p in pods) or all(p < 0 for p in pods)
        if pods[0] >= 0:
            assert len({int(lv[2][p]) for p in pods}) == 1
    # the hint annotation carries the pod names
    tmpl = {}
    mgr.InjectPodGroupLabels(lws_group("a", 1, RACK, lws=4), tmpl)
    assert "a-decode-0-0" in tmpl["metadata"]["annotations"]["rbg.workloads.x-k8s.io/b200-topo-placement"]


def test_colocation_without_exclusive_keys_is_level_0():
    topo, _ = topo_and_levels()
    pl = LwPlacer(topo)
    mgr = B200TopoPodGroupManager(pl, leader_worker=True)
    mgr.reconcile_pod_groups([lws_group("a", 1, "anything")])
    assert pl.lw_calls[0].tolist() == [[2, 0], [1, -1]]


def test_no_hint_reasons():
    topo, lv = topo_and_levels()
    pl = LwPlacer(topo, lv[:2])      # the snapshot holds level 1 only
    mgr = B200TopoPodGroupManager(pl, exclusive_keys=[NV, HOSTNAME, RACK], leader_worker=True)
    out = mgr.reconcile_pod_groups([lws_group("unknown", 1, "example.com/row"), lws_group("missing", 2, RACK),
                                    lws_group("ok", 3, HOSTNAME), plain_group("p", 4)])
    assert [p.status for p in out][:2] == [RBGTOPO_NO_HINT] * 2 and out[2].status != RBGTOPO_NO_HINT
    assert "not configured" in mgr.no_hint[("ns", "unknown")]
    assert "no level 2" in mgr.no_hint[("ns", "missing")]
    out = mgr.reconcile_pod_groups([lws_group("x", 5), plain_group("p", 4)], committed=True)
    assert out[0].status == RBGTOPO_NO_HINT and "committed" in mgr.no_hint[("ns", "x")]
    assert out[1].status != RBGTOPO_NO_HINT
    ranked = B200TopoPodGroupManager(pl, alternates=2, leader_worker=True)
    out = ranked.reconcile_pod_groups([lws_group("y", 6)])
    assert out[0].status == RBGTOPO_NO_HINT and "alternates" in ranked.no_hint[("ns", "y")]


def test_leader_worker_off_leaves_everything_as_it_was():
    topo, _ = topo_and_levels()
    groups = [lws_group("a", 1, "anything", lws=4), plain_group("b", 2)]
    pl_off, pl_on = LwPlacer(topo), LwPlacer(topo)
    off = B200TopoPodGroupManager(pl_off).reconcile_pod_groups(groups)
    assert not pl_off.lw_calls and pl_off.plain_calls == 1
    assert set(off[0].nodes) == {"a-decode-0", "a-decode-1", "a-router-0"}
    # groups without a multi-pod role never take the leader-worker call
    on = B200TopoPodGroupManager(pl_on, leader_worker=True).reconcile_pod_groups(groups[1:])
    assert not pl_on.lw_calls
    assert [(p.status, p.nodes, p.domain) for p in on] == [(p.status, p.nodes, p.domain) for p in off[1:]]


def test_the_same_group_twice_gets_two_results_in_order():
    topo, _ = topo_and_levels()
    a, b = lws_group("a", 1), plain_group("b", 2)
    out = B200TopoPodGroupManager(LwPlacer(topo), leader_worker=True).reconcile_pod_groups([a, b, a, b])
    assert [set(p.nodes) for p in out[:2]] == [set(p.nodes) for p in out[2:]]
    assert all(k.startswith("a-") for k in out[0].nodes) and all(k.startswith("b-") for k in out[1].nodes)
