"""The plugin mirror with node classes in committed batches (rbg_b200/plugin.py, DESIGN.md §3.20): a committed batch
that holds a restricted group goes through ONE place_groups_eligible_committed call (ranked with alternates) in the
given order — masks for every role, all ones for unrestricted groups, role_pods only when a leader-worker group is in
the batch, pod-keyed hints for such groups — and every hint and alternate lands on a node its role admits; batches of
unrestricted groups place exactly as before; the remaining no-hint reasons stay.  On CPU the placer behind the manager
is the oracle (tests/eligible_committed_oracle.py); the GPU test runs a committed mooncake batch through the C ABI."""
import dataclasses

import numpy as np
import pytest

from eligible_committed_oracle import run_eligible_committed, run_eligible_committed_ranked
from lw_committed_oracle import run_lw_committed
from rbg_b200 import synth
from rbg_b200.engine import TopoPlacer
from rbg_b200.ingest import NodeIndex, NodeInfo, build_node_classes
from rbg_b200.plugin import ALL_CLASSES, RBGTOPO_NO_HINT, B200TopoPodGroupManager
from test_plugin_eligible import (GPU_TAINT, TOLERATE_GPU, OraclePlacer, admitted, cpu_roles, gpu_group, snapshot,
                                  unrestricted)


class CommittedPlacer(OraclePlacer):
    """OraclePlacer plus committed batches of any length and place_groups_eligible_committed[_ranked]."""

    def __init__(self, topo, classes, **kw):
        super().__init__(topo, classes, **kw)
        self.places_eligible_committed = self.world == 1

    def place_groups_committed(self, gb):
        self.calls.append("place_groups_committed")
        return (*run_lw_committed(self.topo, gb, self._rp(gb)), 1)

    def place_groups_lw_committed(self, gb, rp):
        self.calls.append("place_groups_lw_committed")
        return (*run_lw_committed(self.topo, gb, rp), 1)

    def place_groups_eligible_committed(self, gb, rp, masks):
        self.calls.append(("place_groups_eligible_committed", None if rp is None else [tuple(x) for x in rp],
                           [int(m) for m in masks]))
        return (*run_eligible_committed(self.topo, gb, rp, masks, self.cls), 1)

    def place_groups_eligible_committed_ranked(self, gb, rp, masks, n_alt):
        self.calls.append(("place_groups_eligible_committed_ranked", None if rp is None else [tuple(x) for x in rp],
                           [int(m) for m in masks]))
        a, s, d, sc, an, asc = run_eligible_committed_ranked(self.topo, gb, rp, masks, self.cls, n_alt)
        return a, s, d, 1, sc, an, asc


def role_of(rbg, key):
    """The role of hint key "{rbg}-{role}-{ordinal}[-{k}]" (role names may hold hyphens)."""
    rest = key[len(rbg.name) + 1:]
    return max((r for r in rbg.roles if rest.startswith(r.name + "-")), key=lambda r: len(r.name))


def check_admitted(classes, rbg, placement):
    for key, node in placement.nodes.items():
        role = role_of(rbg, key)
        if node >= 0:
            assert admitted(classes, role, node), (key, node)
        for alt in placement.alternates.get(key, []):
            assert admitted(classes, role, alt), (key, alt)


def _masks(classes, rbg):
    from rbg_b200.ingest import role_admit
    return [role_admit(classes, r.node_selector, r.node_affinity, r.tolerations) for r in rbg.roles]


@pytest.mark.parametrize("alternates", [0, 3])
def test_one_call_for_the_whole_batch(alternates):
    topo, classes = snapshot()
    pl = CommittedPlacer(topo, classes)
    mgr = B200TopoPodGroupManager(pl, alternates=alternates, node_classes=classes)
    rbgs = [cpu_roles(), gpu_group(), unrestricted(), cpu_roles("svc2", 4)]
    out = mgr.reconcile_pod_groups(rbgs, committed=True)
    assert len(pl.calls) == 1
    name, rp, masks = pl.calls[0]
    assert name == ("place_groups_eligible_committed_ranked" if alternates else "place_groups_eligible_committed")
    assert rp is None   # no leader-worker group: role_pods NULL
    runs = mgr.groups_blob(rbgs)[1]
    want = [(_masks(classes, g.rbg) if mgr.is_restricted(g.rbg) else [ALL_CLASSES] * len(g.rbg.roles))[ri]
            for g in runs for ri in g.order]
    assert masks == want and ALL_CLASSES in masks
    for rbg, p in zip(rbgs, out):
        assert p.status != RBGTOPO_NO_HINT and all(v >= 0 for v in p.nodes.values())
        check_admitted(classes, rbg, p)
    # the batch is committed: the two CPU-only groups do not both take the last room of a node
    used = {}
    for rbg, p in zip(rbgs, out):
        for key, node in p.nodes.items():
            role = role_of(rbg, key)
            used[node] = used.get(node, 0) + role.demand
    assert all(used[n] <= topo.free[n] for n in used)
    if alternates:
        assert any(out[0].alternates.values())


def test_leader_worker_groups_get_pod_keyed_hints_and_role_pods():
    topo, classes = snapshot()
    pl = CommittedPlacer(topo, classes)
    mgr = B200TopoPodGroupManager(pl, alternates=2, leader_worker=True, node_classes=classes)
    rbgs = [gpu_group(lws=2), cpu_roles()]
    p = mgr.reconcile_pod_groups(rbgs, committed=True)
    assert len(pl.calls) == 1 and pl.calls[0][0] == "place_groups_eligible_committed_ranked"
    runs = mgr.groups_blob(rbgs)[1]
    want = [((2, -1) if g.rbg.name == "serve" and g.rbg.roles[ri].name == "prefill" else (1, -1))
            for g in runs for ri in g.order]
    assert pl.calls[0][1] == want   # (S, C) for every role, (1, -1) for standalone roles
    assert sorted(p[0].nodes) == ["serve-prefill-0-0", "serve-prefill-0-1", "serve-prefill-1-0", "serve-prefill-1-1",
                                  "serve-router-0"]
    assert all(v >= 0 for q in p for v in q.nodes.values())
    check_admitted(classes, rbgs[0], p[0])
    check_admitted(classes, rbgs[1], p[1])


def test_unrestricted_batches_place_as_before():
    topo, classes = snapshot()
    rbgs = [unrestricted("u1", 3), unrestricted("u2", 4)]
    with_cls = B200TopoPodGroupManager(CommittedPlacer(topo, classes), node_classes=classes)
    without = B200TopoPodGroupManager(CommittedPlacer(topo, classes))
    a = with_cls.reconcile_pod_groups(rbgs, committed=True)
    b = without.reconcile_pod_groups(rbgs, committed=True)
    assert [(p.status, p.nodes, p.domain) for p in a] == [(p.status, p.nodes, p.domain) for p in b]
    assert with_cls.placer.calls == ["place_groups_committed"]


def test_remaining_no_hint_reasons():
    topo, classes = snapshot()
    cases = [
        (OraclePlacer(topo, classes), "committed batches place no node classes"),        # no such call
        (CommittedPlacer(topo, classes, world=2), "committed batches place no node classes"),
    ]
    for pl, text in cases:
        mgr = B200TopoPodGroupManager(pl, node_classes=classes)
        out = mgr.reconcile_pod_groups([cpu_roles(), unrestricted()], committed=True)
        assert out[0].status == RBGTOPO_NO_HINT and text in mgr.no_hint[("default", "svc")], mgr.no_hint
    # an undecidable selector keeps its own reason; the decidable restricted group still gets its hint
    mgr = B200TopoPodGroupManager(CommittedPlacer(topo, classes), node_classes=classes)
    out = mgr.reconcile_pod_groups([gpu_group(selector={"zone": "a"}), cpu_roles()], committed=True)
    assert out[0].status == RBGTOPO_NO_HINT and "'zone'" in mgr.no_hint[("default", "serve")]
    assert out[1].status != RBGTOPO_NO_HINT
    # a group at an exclusive level >= 1 on a placer without committed leader-worker levels
    pl = CommittedPlacer(topo, classes)
    pl.places_levels = pl.places_committed_levels = True
    pl._n_levels = 1
    mgr = B200TopoPodGroupManager(pl, exclusive_keys=("d", "rack"), node_classes=classes)
    lv = unrestricted("lv", 5)
    lv.annotations["rbg.workloads.x-k8s.io/group-exclusive-topology"] = "rack"
    out = mgr.reconcile_pod_groups([cpu_roles(), lv], committed=True)
    assert out[0].status == RBGTOPO_NO_HINT and "committed batches place no node classes" in mgr.no_hint[("default", "svc")]
    assert not any(isinstance(c, tuple) for c in pl.calls)
    # the step-batch path
    mgr = B200TopoPodGroupManager(CommittedPlacer(topo, classes), node_classes=classes)
    assert mgr.reconcile_pod_groups_by_waves([cpu_roles()])[0].status == RBGTOPO_NO_HINT
    assert "step-batch" in mgr.no_hint[("default", "svc")]


def _mooncake_batch(n_groups, n):
    import bench
    gpu_roles = {"mooncake-store", "prefill", "decode"}
    out = []
    for rbg in bench.to_plugin(bench.fleet_spec("mooncake", n_groups, n, 3)):
        rbg.roles = [dataclasses.replace(r, tolerations=TOLERATE_GPU) if r.name in gpu_roles else r for r in rbg.roles]
        out.append(rbg)
    return out


def _tainted(n):
    """Two thirds of the nodes are GPU nodes tainted NoSchedule; the rest are the CPU pool."""
    topo = synth.make_topology(n, seed=9, tiers=2, max_free=4)
    topo.domain_owner = np.full(int(topo.domain.max()) + 1, -1, np.int32)
    nodes = [NodeInfo(name=f"node-{k:04d}", labels={"pool": "cpu" if k % 3 == 0 else "gpu"},
                      taints=[] if k % 3 == 0 else [GPU_TAINT]) for k in range(n)]
    return topo, build_node_classes(nodes, NodeIndex([nd.name for nd in nodes], ["d"]), ("pool",))


def test_committed_mooncake_batch_on_the_oracle():
    topo, classes = _tainted(256)
    rbgs = _mooncake_batch(6, 256)
    mgr = B200TopoPodGroupManager(CommittedPlacer(topo, classes), alternates=2, node_classes=classes)
    out = mgr.reconcile_pod_groups(rbgs, committed=True)
    assert all(p.status != RBGTOPO_NO_HINT for p in out)
    for rbg, p in zip(rbgs, out):
        check_admitted(classes, rbg, p)


@pytest.mark.gpu
def test_committed_mooncake_batch_on_the_device():
    """A committed mooncake batch on a cluster whose GPU nodes are tainted: a hint for every group, no router or master
    on a GPU node, and the same hints and alternates as the CPU placer gives."""
    n = 1024
    topo, classes = _tainted(n)
    rbgs = _mooncake_batch(10, n)
    eng = TopoPlacer(device=0)
    try:
        eng.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
        eng.set_node_classes(classes.node_class, classes.n_classes)
        out = B200TopoPodGroupManager(eng, alternates=3, node_classes=classes).reconcile_pod_groups(rbgs, committed=True)
        exp = B200TopoPodGroupManager(CommittedPlacer(topo, classes), alternates=3,
                                      node_classes=classes).reconcile_pod_groups(rbgs, committed=True)
        for rbg, p, e in zip(rbgs, out, exp):
            assert p.status != RBGTOPO_NO_HINT
            assert (p.status, p.nodes, p.domain, p.alternates) == (e.status, e.nodes, e.domain, e.alternates)
            check_admitted(classes, rbg, p)
            for key, node in p.nodes.items():
                if key.startswith(f"{rbg.name}-router-") or key.startswith(f"{rbg.name}-mooncake-master-"):
                    assert node < 0 or classes.labels[classes.node_class[node]]["pool"] == "cpu", (key, node)
    finally:
        eng.close()
