"""The plugin mirror with node classes (rbg_b200/plugin.py, DESIGN.md §3.19): a group whose role templates exclude an
installed class is placed through place_groups_eligible (ranked with alternates, with its (S, C) table and pod-keyed
hints when it runs leader-worker replicas), and every hint and alternate lands on a node its role admits; committed
batches, world > 1, a placer without the call, the step-batch path and undecidable selectors give no hint and a
reason; unrestricted groups place exactly as under a manager without node_classes.  On CPU the placer behind the
manager is the oracle (tests/eligible_oracle.py, tests/lw_oracle.py); the GPU test runs the same through the C ABI."""
import numpy as np
import pytest

import lw_oracle as lw
from eligible_oracle import run_eligible, run_eligible_ranked
from lw_alternates_oracle import run_lw_ranked
from rbg_b200 import synth
from rbg_b200.engine import TopoPlacer
from rbg_b200.ingest import NodeIndex, NodeInfo, build_node_classes
from rbg_b200.plugin import RBGTOPO_NO_HINT, B200TopoPodGroupManager, RoleBasedGroup, RoleSpec

N = 96
GPU_TAINT = {"key": "nvidia.com/gpu", "value": "present", "effect": "NoSchedule"}
TOLERATE_GPU = [{"key": "nvidia.com/gpu", "operator": "Exists"}]


def snapshot():
    """A third of the nodes is the CPU pool; the rest are tainted GPU nodes of two pools."""
    topo = synth.make_topology(N, seed=9, tiers=2, max_free=4)
    topo.domain_owner = np.full(int(topo.domain.max()) + 1, -1, np.int32)
    nodes = [NodeInfo(name=f"node-{n:03d}", labels={"pool": ("cpu", "h100", "a100")[n % 3]},
                      taints=[] if n % 3 == 0 else [GPU_TAINT]) for n in range(N)]
    index = NodeIndex([nd.name for nd in nodes], ["d"])
    return topo, build_node_classes(nodes, index, ("pool",))


class OraclePlacer:
    """place_groups[_ranked], place_groups_lw[_ranked] and place_groups_eligible[_ranked] from the CPU oracles."""

    def __init__(self, topo, classes, world=1, places_eligible=True):
        self.topo, self.n_nodes, self.world, self.places_eligible = topo, topo.n, world, places_eligible
        self.places_lw_ranked = True
        self.cls = classes.node_class
        self.calls = []

    def _rp(self, gb):
        return lw.role_pods_for(gb, lambda g, r: (1, -1))

    def place_groups(self, gb):
        self.calls.append("place_groups")
        return lw.run_lw(self.topo, gb, self._rp(gb))

    def place_groups_committed(self, gb):   # the tests commit batches of one group: the snapshot placement
        assert int(gb[2]) == 1
        return (*self.place_groups(gb), 1)

    def place_groups_ranked(self, gb, n_alt):
        self.calls.append("place_groups_ranked")
        return run_lw_ranked(self.topo, gb, self._rp(gb), n_alt)

    def place_groups_lw(self, gb, rp):
        self.calls.append("place_groups_lw")
        return lw.run_lw(self.topo, gb, rp)

    def place_groups_lw_ranked(self, gb, rp, n_alt):
        self.calls.append("place_groups_lw_ranked")
        return run_lw_ranked(self.topo, gb, rp, n_alt)

    def place_groups_eligible(self, gb, rp, masks):
        self.calls.append(("place_groups_eligible", rp is None, [int(m) for m in masks]))
        return run_eligible(self.topo, gb, rp, masks, self.cls)

    def place_groups_eligible_ranked(self, gb, rp, masks, n_alt):
        self.calls.append(("place_groups_eligible_ranked", rp is None, [int(m) for m in masks]))
        return run_eligible_ranked(self.topo, gb, rp, masks, self.cls, n_alt)


def cpu_roles(name="svc", gid=1):
    """The mooncake router / master shape: demand 0, no toleration for the GPU taint."""
    return RoleBasedGroup("default", name, [RoleSpec("router", 2, (), 0), RoleSpec("master", 1, (), 0)], gid=gid)


def gpu_group(name="serve", gid=2, lws=0, selector=None):
    return RoleBasedGroup("default", name, [
        RoleSpec("prefill", 2, (), 1, lws_size=lws, node_selector=selector or {"pool": "h100"},
                 tolerations=TOLERATE_GPU),
        RoleSpec("router", 1, ("prefill",), 0)], gid=gid)


def unrestricted(name="free", gid=3):
    tol = [{"operator": "Exists"}]
    return RoleBasedGroup("default", name, [RoleSpec("a", 2, (), 1, tolerations=tol),
                                            RoleSpec("b", 1, ("a",), 1, tolerations=tol)], gid=gid)


def admitted(classes, role, node):
    from rbg_b200.ingest import role_admit
    mask = role_admit(classes, role.node_selector, role.node_affinity, role.tolerations)
    return (mask >> int(classes.node_class[node])) & 1


def check_admitted(classes, rbg, placement):
    roles = {r.name: r for r in rbg.roles}
    for key, node in placement.nodes.items():
        role = roles[key[len(rbg.name) + 1:].split("-")[0]]
        if node >= 0:
            assert admitted(classes, role, node), (key, node)
        for alt in placement.alternates.get(key, []):
            assert admitted(classes, role, alt), (key, alt)


@pytest.mark.parametrize("alternates", [0, 3])
def test_restricted_groups_route_through_the_eligible_call(alternates):
    topo, classes = snapshot()
    pl = OraclePlacer(topo, classes)
    mgr = B200TopoPodGroupManager(pl, alternates=alternates, node_classes=classes)
    rbgs = [cpu_roles(), gpu_group(), unrestricted()]
    out = mgr.reconcile_pod_groups(rbgs)
    name = "place_groups_eligible_ranked" if alternates else "place_groups_eligible"
    elig = [c for c in pl.calls if isinstance(c, tuple)]
    assert len(elig) == 1 and elig[0][0] == name and elig[0][1]   # one call, no leader-worker group: role_pods NULL
    assert ("place_groups_ranked" if alternates else "place_groups") in pl.calls
    for rbg, p in zip(rbgs, out):
        assert p.status != RBGTOPO_NO_HINT and all(v >= 0 for v in p.nodes.values())
        check_admitted(classes, rbg, p)
    # the CPU-only roles stay in the CPU pool, although GPU nodes outrank them without classes
    assert all(classes.labels[classes.node_class[v]]["pool"] == "cpu" for v in out[0].nodes.values())
    bare = B200TopoPodGroupManager(OraclePlacer(topo, classes), alternates=alternates).reconcile_pod_groups([cpu_roles()])
    assert any(classes.labels[classes.node_class[v]]["pool"] != "cpu" for v in bare[0].nodes.values())
    if alternates:
        assert any(out[0].alternates.values())


def test_unrestricted_groups_place_as_without_node_classes():
    topo, classes = snapshot()
    rbgs = [unrestricted("u1", 3), unrestricted("u2", 4)]
    with_cls = B200TopoPodGroupManager(OraclePlacer(topo, classes), alternates=2, node_classes=classes)
    without = B200TopoPodGroupManager(OraclePlacer(topo, classes), alternates=2)
    a, b = with_cls.reconcile_pod_groups(rbgs), without.reconcile_pod_groups(rbgs)
    assert [(p.status, p.nodes, p.domain, p.alternates) for p in a] == [(p.status, p.nodes, p.domain, p.alternates)
                                                                        for p in b]
    assert not any(isinstance(c, tuple) for c in with_cls.placer.calls)


def test_leader_worker_groups_get_pod_keyed_hints():
    topo, classes = snapshot()
    pl = OraclePlacer(topo, classes)
    mgr = B200TopoPodGroupManager(pl, alternates=2, leader_worker=True, node_classes=classes)
    rbg = gpu_group(lws=2)
    p = mgr.reconcile_pod_groups([rbg, cpu_roles()])
    elig = [c for c in pl.calls if isinstance(c, tuple)]
    assert len(elig) == 1 and not elig[0][1]   # role_pods given
    assert sorted(p[0].nodes) == ["serve-prefill-0-0", "serve-prefill-0-1", "serve-prefill-1-0", "serve-prefill-1-1",
                                  "serve-router-0"]
    assert all(v >= 0 for v in p[0].nodes.values())
    check_admitted(classes, rbg, p[0])
    check_admitted(classes, cpu_roles(), p[1])


def test_no_hint_reasons():
    topo, classes = snapshot()
    cases = [
        (dict(), dict(committed=True), "committed"),
        (dict(world=2), dict(), "world > 1"),
        (dict(places_eligible=False), dict(), "no rbgtopo_place_groups_eligible"),
    ]
    for pkw, ckw, text in cases:
        mgr = B200TopoPodGroupManager(OraclePlacer(topo, classes, **pkw), node_classes=classes)
        out = mgr.reconcile_pod_groups([cpu_roles(), unrestricted()], **ckw)
        assert out[0].status == RBGTOPO_NO_HINT and text in mgr.no_hint[("default", "svc")], mgr.no_hint
        assert out[1].status != RBGTOPO_NO_HINT and ("default", "free") not in mgr.no_hint
    mgr = B200TopoPodGroupManager(OraclePlacer(topo, classes), node_classes=classes)
    out = mgr.reconcile_pod_groups([gpu_group(selector={"zone": "a"})])
    assert out[0].status == RBGTOPO_NO_HINT and "'zone'" in mgr.no_hint[("default", "serve")]
    aff = RoleBasedGroup("default", "mf", [RoleSpec("x", 1, (), 1, tolerations=TOLERATE_GPU, node_affinity=[
        {"matchFields": [{"key": "metadata.name", "operator": "In", "values": ["node-001"]}]}])], gid=7)
    assert mgr.reconcile_pod_groups([aff])[0].status == RBGTOPO_NO_HINT and "matchFields" in mgr.no_hint[("default", "mf")]
    assert mgr.reconcile_pod_groups_by_waves([cpu_roles()])[0].status == RBGTOPO_NO_HINT
    assert "step-batch" in mgr.no_hint[("default", "svc")]


@pytest.mark.gpu
def test_on_the_device():
    """The same routing through TopoPlacer: restricted hints equal the engine's eligible call, every hint admitted,
    unrestricted groups as under a manager without node_classes."""
    topo, classes = snapshot()
    eng = TopoPlacer(device=0)
    try:
        eng.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
        eng.set_node_classes(classes.node_class, classes.n_classes)
        rbgs = [cpu_roles(), gpu_group(lws=2), unrestricted()]
        mgr = B200TopoPodGroupManager(eng, alternates=3, leader_worker=True, node_classes=classes)
        out = mgr.reconcile_pod_groups(rbgs)
        cpu = OraclePlacer(topo, classes)
        exp = B200TopoPodGroupManager(cpu, alternates=3, leader_worker=True, node_classes=classes).reconcile_pod_groups(rbgs)
        for rbg, p, e in zip(rbgs, out, exp):
            assert (p.status, p.nodes, p.domain, p.alternates) == (e.status, e.nodes, e.domain, e.alternates)
            check_admitted(classes, rbg, p)
        bare = B200TopoPodGroupManager(eng, alternates=3, leader_worker=True).reconcile_pod_groups([unrestricted()])
        assert (bare[0].nodes, bare[0].alternates) == (out[2].nodes, out[2].alternates)
    finally:
        eng.close()
