"""Node-topology ingestion (SURVEY.md §8f rank 1): Node objects -> the snapshot arrays of
rbgtopo_set_topology / rbgtopo_update_nodes.

The reference has no Node informer (SURVEY.md §0: the controller never lists Nodes; RBAC for
`nodes` would be new, cf. cmd/rbgs/main.go:408-429 cache options).  This is the Python mirror of
the `nodeCache` the Go shim of INTEGRATION.md §2 keeps: node labels name the tier groups a node
belongs to, closest tier first, and two nodes are linked with the weight of the closest tier
they share (NVLink domain 1000 > host / PCIe group 100 > RDMA leaf 10 > zone / VPC 1 — the
README.md:53 order of the reference, spec §3.1).

Determinism (placements must not depend on informer event order): nodes are numbered by name,
groups by label value; inside a tier group every node links to its `fanout[tier]` successors in
name order (cyclically; the whole group when it is small enough), which yields a symmetric,
duplicate-free CSR with sorted rows — what rbgtopo_set_topology validates.
"""
from __future__ import annotations

import re
from dataclasses import dataclass, field
from typing import Dict, List, Mapping, Optional, Sequence, Tuple

import numpy as np

from .synth import TIER_W, Topology

# label conventions of the shim (closest tier first); the first one is also the exclusive-topology
# domain (rbg.workloads.x-k8s.io/group-exclusive-topology names a topology key, annotation.go:25)
DEFAULT_TIER_LABELS: Tuple[str, ...] = (
    "nvidia.com/nvlink-domain",            # NVL72 / NVSwitch domain
    "kubernetes.io/hostname-group",        # hosts behind one PCIe / NIC complex
    "network.topology/rdma-leaf",          # RDMA leaf switch
    "topology.kubernetes.io/zone",         # VPC / zone
)
DEFAULT_FANOUT: Tuple[int, ...] = (71, 8, 8, 4)    # links per node and tier (whole NVL72 domain; samples above)
ACCELERATOR_RESOURCE = "nvidia.com/gpu"
MAX_FREE = 32767                                   # RBGTOPO_MAX_FREE


@dataclass
class NodeInfo:
    """The fields of corev1.Node this path reads."""
    name: str
    labels: Mapping[str, str] = field(default_factory=dict)
    allocatable: Mapping[str, int] = field(default_factory=dict)   # resource -> count
    requested: Mapping[str, int] = field(default_factory=dict)     # summed over the node's pods
    unschedulable: bool = False                                    # spec.unschedulable / not Ready
    taints: Sequence[Mapping[str, str]] = ()                       # spec.taints: {key, value, effect}


@dataclass
class NodeIndex:
    """Node name <-> dense id and domain name <-> dense id of one snapshot (hints are written back
    with these: Placement.nodes holds ids)."""
    names: List[str]
    domains: List[str]

    def node_id(self, name: str) -> int:
        return self._ids[name]

    def __post_init__(self):
        self._ids: Dict[str, int] = {nm: i for i, nm in enumerate(self.names)}


def free_slots(node: NodeInfo, resource: str = ACCELERATOR_RESOURCE) -> int:
    if node.unschedulable:
        return 0
    return int(max(0, min(MAX_FREE, node.allocatable.get(resource, 0) - node.requested.get(resource, 0))))


def build_topology(nodes: Sequence[NodeInfo], tier_labels: Sequence[str] = DEFAULT_TIER_LABELS,
                   fanout: Sequence[int] = DEFAULT_FANOUT, resource: str = ACCELERATOR_RESOURCE,
                   domain_owner: Optional[Mapping[str, int]] = None) -> Tuple[Topology, NodeIndex]:
    """Snapshot arrays for rbgtopo_set_topology.  `domain_owner`: domain name -> gid of the group
    that occupies it exclusively (pods carrying the exclusive-topology affinity,
    pkg/reconciler/pod_reconciler.go:192-229); absent = free."""
    if len(tier_labels) > len(TIER_W) or len(fanout) < len(tier_labels):
        raise ValueError("at most 4 tiers, one fanout per tier")
    order = sorted(range(len(nodes)), key=lambda i: nodes[i].name)
    names = [nodes[i].name for i in order]
    if len(set(names)) != len(names):
        raise ValueError("duplicate node name")
    n = len(names)
    src: List[np.ndarray] = []
    dst: List[np.ndarray] = []
    wts: List[np.ndarray] = []
    for tier, key in enumerate(tier_labels):
        groups: Dict[str, List[int]] = {}
        for new_id, i in enumerate(order):
            v = nodes[i].labels.get(key)
            if v is not None:
                groups.setdefault(v, []).append(new_id)
        for members in groups.values():          # members are ascending ids = name order
            m = len(members)
            if m < 2:
                continue
            k = min(fanout[tier], m - 1)
            ids = np.asarray(members, dtype=np.int64)
            for off in range(1, k + 1):
                peer = np.roll(ids, -off)
                src.append(ids); dst.append(peer)
                src.append(peer); dst.append(ids)
                wts.append(np.full(2 * m, TIER_W[tier], dtype=np.int64))
    if src:
        a = np.concatenate(src); b = np.concatenate(dst); w = np.concatenate(wts)
        keep = a != b
        a, b, w = a[keep], b[keep], w[keep]
        # a pair keeps its closest tier = largest weight: sort by (a, b, -w), take the first of each pair
        o = np.lexsort((-w, b, a))
        a, b, w = a[o], b[o], w[o]
        first = np.ones(len(a), dtype=bool)
        first[1:] = (a[1:] != a[:-1]) | (b[1:] != b[:-1])
        a, b, w = a[first], b[first], w[first]
    else:
        a = b = w = np.zeros(0, dtype=np.int64)
    row_ptr = np.zeros(n + 1, dtype=np.int64)
    np.add.at(row_ptr, a + 1, 1)
    row_ptr = np.cumsum(row_ptr)
    # exclusive-topology domain = group of the closest tier; nodes without the label get a domain of their own
    dom_names: List[str] = []
    dom_id: Dict[str, int] = {}
    domain = np.zeros(n, dtype=np.int32)
    for new_id, i in enumerate(order):
        v = nodes[i].labels.get(tier_labels[0]) if tier_labels else None
        key = v if v is not None else f"node/{names[new_id]}"
        if key not in dom_id:
            dom_id[key] = len(dom_names)
            dom_names.append(key)
        domain[new_id] = dom_id[key]
    owner = np.full(max(1, len(dom_names)), -1, dtype=np.int32)
    for dname, gid in (domain_owner or {}).items():
        if dname in dom_id:
            owner[dom_id[dname]] = gid
    free = np.asarray([free_slots(nodes[i], resource) for i in order], dtype=np.int32)
    topo = Topology(row_ptr.astype(np.int32), b.astype(np.int32), w.astype(np.int32), free, domain, owner)
    return topo, NodeIndex(names, dom_names)


def refresh(topo: Topology, index: NodeIndex, nodes: Sequence[NodeInfo], resource: str = ACCELERATOR_RESOURCE,
            domain_owner: Optional[Mapping[str, int]] = None) -> Tuple[np.ndarray, np.ndarray]:
    """(free, domain_owner) for rbgtopo_update_nodes from fresh Node objects of the SAME node set
    (capacity / ownership churn).  Node add / remove changes the CSR: call build_topology."""
    by_name = {nd.name: nd for nd in nodes}
    if set(by_name) != set(index.names):
        raise ValueError("node set changed: rebuild the topology")
    free = np.asarray([free_slots(by_name[nm], resource) for nm in index.names], dtype=np.int32)
    owner = np.full(len(topo.domain_owner), -1, dtype=np.int32)
    for dname, gid in (domain_owner or {}).items():
        if dname in index.domains:
            owner[index.domains.index(dname)] = gid
    return free, owner


@dataclass
class ExclusiveLevels:
    """Node partitions of the exclusive-topology keys (DESIGN.md §3.9): keys[0] is the level-0 label (the domain of
    build_topology), keys[L] for L >= 1 gives domain[L - 1][n] with n_domains[L - 1] domains named names[L - 1]."""
    keys: Tuple[str, ...]
    domain: np.ndarray                 # [len(keys) - 1][n] int32
    n_domains: np.ndarray              # [len(keys) - 1] int32
    names: List[List[str]]


def build_exclusive_levels(nodes: Sequence[NodeInfo], index: NodeIndex, keys: Sequence[str]) -> ExclusiveLevels:
    """Partitions for rbgtopo_set_exclusive_levels, node ids of `index` (build_topology).  As for level 0, a node
    without the label gets a domain of its own, and domain ids follow node-name order, so the result does not depend
    on the order the informer delivered the nodes in."""
    if not keys:
        raise ValueError("keys[0] must be the level-0 label")
    by_name = {nd.name: nd for nd in nodes}
    if set(by_name) != set(index.names):
        raise ValueError("node set changed: rebuild the topology")
    rows, counts, names = [], [], []
    for key in keys[1:]:
        ids: Dict[str, int] = {}
        row = np.zeros(len(index.names), dtype=np.int32)
        for n, nm in enumerate(index.names):        # index.names is name-sorted
            v = by_name[nm].labels.get(key)
            k = v if v is not None else f"node/{nm}"
            row[n] = ids.setdefault(k, len(ids))
        rows.append(row)
        counts.append(max(1, len(ids)))
        names.append(list(ids))
    dom = np.stack(rows) if rows else np.zeros((0, len(index.names)), dtype=np.int32)
    return ExclusiveLevels(tuple(keys), dom, np.asarray(counts, dtype=np.int32), names)


def exclusive_occupancy(levels: ExclusiveLevels, index: NodeIndex,
                        pods: Sequence[Tuple[str, int, str]]) -> np.ndarray:
    """Records (node, gid, level) for rbgtopo_set_exclusive_levels from the pods that carry the group-unique-hash
    label: (node name, gid of the pod's group, the topology key its group's annotation names).  Pods on nodes
    outside the snapshot are skipped; a key outside `levels.keys` is an error (that group cannot be placed)."""
    pos = {nm: i for i, nm in enumerate(index.names)}
    out = []
    for node, gid, key in pods:
        if node not in pos:
            continue
        if key not in levels.keys:
            raise ValueError(f"exclusive key {key!r} is not configured")
        out.append((pos[node], int(gid), levels.keys.index(key)))
    out.sort()
    return np.asarray(out, dtype=np.int32).reshape(-1, 3)


# ---- node classes (DESIGN.md §3.19) ----------------------------------------------------------------------------------
# Only these taint effects keep a pod off a node; PreferNoSchedule is a preference and is ignored.
HARD_TAINT_EFFECTS = ("NoSchedule", "NoExecute")
MAX_NODE_CLASSES = 64   # RBGTOPO_MAX_NODE_CLASSES


@dataclass
class NodeClasses:
    """Classes for rbgtopo_set_node_classes: node_class[n] (node ids of `index`), and per class the values of the
    configured label keys (a missing label is absent) and its NoSchedule / NoExecute taints as (key, value, effect)."""
    keys: Tuple[str, ...]
    node_class: np.ndarray                       # [n] int32
    labels: List[Dict[str, str]]
    taints: List[Tuple[Tuple[str, str, str], ...]]

    @property
    def n_classes(self) -> int:
        return len(self.labels)


class NotDecidable(ValueError):
    """A selector the classes cannot decide (a label key outside the configured keys, or matchFields): the group
    gets no hint."""


def build_node_classes(nodes: Sequence[NodeInfo], index: NodeIndex, keys: Sequence[str]) -> NodeClasses:
    """Nodes with the same values of `keys` and the same hard taints share a class.  Classes are numbered by first
    appearance over the name-sorted nodes of `index`, so the result does not depend on informer order.  More than
    RBGTOPO_MAX_NODE_CLASSES (64) classes is an error."""
    by_name = {nd.name: nd for nd in nodes}
    if set(by_name) != set(index.names):
        raise ValueError("node set changed: rebuild the topology")
    ids: Dict[tuple, int] = {}
    cls = np.zeros(len(index.names), dtype=np.int32)
    for n, nm in enumerate(index.names):
        nd = by_name[nm]
        lab = tuple((k, nd.labels[k]) for k in keys if k in nd.labels)
        tnt = tuple(sorted({(t.get("key", ""), t.get("value", ""), t.get("effect", "")) for t in nd.taints
                            if t.get("effect", "") in HARD_TAINT_EFFECTS}))
        cls[n] = ids.setdefault((lab, tnt), len(ids))
    if len(ids) > MAX_NODE_CLASSES:
        raise ValueError(f"{len(ids)} node classes exceed {MAX_NODE_CLASSES}: configure fewer label keys")
    return NodeClasses(tuple(keys), cls, [dict(lab) for lab, _ in ids], [tnt for _, tnt in ids])



def tolerates(tol: Mapping[str, str], taint: Tuple[str, str, str]) -> bool:
    """corev1 Toleration.ToleratesTaint: an empty effect matches every effect, an empty key every key; operator
    Exists matches any value, Equal (or empty) the same value."""
    key, value, effect = taint
    if tol.get("effect", "") and tol.get("effect") != effect:
        return False
    if tol.get("key", "") and tol.get("key") != key:
        return False
    op = tol.get("operator", "") or "Equal"
    if op == "Exists":
        return True
    return op == "Equal" and tol.get("value", "") == value


_INT64 = re.compile(r"[+-]?[0-9]+")


def _int(s) -> Optional[int]:
    """Go's strconv.ParseInt(s, 10, 64): an optional sign and decimal digits only (no spaces, no underscores), within
    int64; None otherwise."""
    s = str(s)
    if not _INT64.fullmatch(s):
        return None
    v = int(s)
    return v if -(1 << 63) <= v < (1 << 63) else None


def _expr_matches(expr: Mapping, labels: Mapping[str, str]) -> bool:
    key, op, values = expr["key"], expr["operator"], list(expr.get("values", ()))
    has = key in labels
    if op == "In":
        return has and labels[key] in values
    if op == "NotIn":
        return not has or labels[key] not in values
    if op == "Exists":
        return has
    if op == "DoesNotExist":
        return not has
    if op in ("Gt", "Lt"):
        if not has or len(values) != 1:
            return False
        a, b = _int(labels[key]), _int(values[0])
        if a is None or b is None:
            return False
        return a > b if op == "Gt" else a < b
    raise ValueError(f"node selector operator {op!r}")


def role_admit(classes: NodeClasses, node_selector: Mapping[str, str] = None, node_affinity: Sequence[Mapping] = (),
               tolerations: Sequence[Mapping[str, str]] = ()) -> int:
    """The class mask of a pod template (bit c: class c admits it), as kube-scheduler's NodeAffinity and
    TaintToleration filters decide: every nodeSelector pair matches, one of the required node-affinity terms
    (node_affinity: the nodeSelectorTerms, ORed; empty = no requirement) has all its matchExpressions match, and every
    NoSchedule / NoExecute taint of the class is tolerated.  Raises NotDecidable for a key outside classes.keys or a
    term with matchFields."""
    node_selector = node_selector or {}
    keys = set(classes.keys)
    for k in node_selector:
        if k not in keys:
            raise NotDecidable(f"nodeSelector key {k!r} is not a configured class key")
    for term in node_affinity:
        if term.get("matchFields"):
            raise NotDecidable("node affinity matchFields cannot be decided per class")
        for e in term.get("matchExpressions", ()):
            if e["key"] not in keys:
                raise NotDecidable(f"node affinity key {e['key']!r} is not a configured class key")
    mask = 0
    for c in range(classes.n_classes):
        lab = classes.labels[c]
        if any(lab.get(k) != v for k, v in node_selector.items()):
            continue
        if node_affinity and not any(term.get("matchExpressions") and
                                     all(_expr_matches(e, lab) for e in term["matchExpressions"])
                                     for term in node_affinity):
            continue
        if all(any(tolerates(t, taint) for t in tolerations) for taint in classes.taints[c]):
            mask |= 1 << c
    return mask
