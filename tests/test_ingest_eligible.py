"""CPU: node classes and role masks from Node and pod-template objects (rbg_b200/ingest.py, DESIGN.md §3.19):
classes do not depend on informer order, tolerations follow corev1 ToleratesTaint, nodeSelector and required node
affinity follow the scheduler's NodeAffinity rules (terms ORed, expressions ANDed, In / NotIn / Exists /
DoesNotExist / Gt / Lt), undecidable selectors are reported, and more than 64 classes is an error."""
import itertools

import numpy as np
import pytest

from rbg_b200.ingest import NodeIndex, NodeInfo, NotDecidable, build_node_classes, role_admit

GPU = {"key": "nvidia.com/gpu", "value": "present", "effect": "NoSchedule"}


def fleet():
    nodes = []
    for i in range(12):
        labels = {"pool": ("h100", "a100", "cpu")[i % 3], "zone": ("a", "b")[i % 2]}
        if i % 4 == 0:
            labels["gen"] = str(8 + i // 4)
        taints = [GPU] if i % 3 != 2 else []
        if i == 5:
            taints = taints + [{"key": "soft", "value": "", "effect": "PreferNoSchedule"}]
        nodes.append(NodeInfo(name=f"n{i:02d}", labels=labels, taints=taints))
    return nodes


def classes_of(nodes, keys=("pool", "zone", "gen")):
    index = NodeIndex(sorted(nd.name for nd in nodes), ["d"])
    return index, build_node_classes(nodes, index, keys)


def admitted(cls, mask):
    return [n for n in range(len(cls.node_class)) if (mask >> int(cls.node_class[n])) & 1]


def test_classes_do_not_depend_on_node_order():
    nodes = fleet()
    _, ref = classes_of(nodes)
    for perm in itertools.islice(itertools.permutations(range(len(nodes))), 0, 200, 37):
        _, got = classes_of([nodes[i] for i in perm])
        assert np.array_equal(got.node_class, ref.node_class) and got.labels == ref.labels
    assert ref.n_classes == len({(nd.labels.get("pool"), nd.labels.get("zone"), nd.labels.get("gen")) for nd in nodes})
    # a PreferNoSchedule taint does not split a class
    assert ref.node_class[5] == ref.node_class[11]


def test_tolerations():
    _, cls = classes_of(fleet())
    cpu_only = admitted(cls, role_admit(cls))
    assert cpu_only == [n for n in range(12) if n % 3 == 2]   # the untainted CPU pool
    everything = list(range(12))
    assert admitted(cls, role_admit(cls, tolerations=[{"operator": "Exists"}])) == everything   # empty key, Exists
    assert admitted(cls, role_admit(cls, tolerations=[{"key": "nvidia.com/gpu", "operator": "Exists"}])) == everything
    assert admitted(cls, role_admit(cls, tolerations=[{"key": "nvidia.com/gpu", "value": "present"}])) == everything
    assert admitted(cls, role_admit(cls, tolerations=[{"key": "nvidia.com/gpu", "operator": "Equal",
                                                       "value": "absent"}])) == cpu_only
    # empty effect matches every effect; a different effect does not
    assert admitted(cls, role_admit(cls, tolerations=[{"key": "nvidia.com/gpu", "operator": "Exists",
                                                       "effect": ""}])) == everything
    assert admitted(cls, role_admit(cls, tolerations=[{"key": "nvidia.com/gpu", "operator": "Exists",
                                                       "effect": "NoExecute"}])) == cpu_only


def test_node_selector_and_affinity_operators():
    nodes = fleet()
    _, cls = classes_of(nodes)
    tol = [{"operator": "Exists"}]

    def sel(**kw):
        return admitted(cls, role_admit(cls, tolerations=tol, **kw))

    lab = [nd.labels for nd in sorted(nodes, key=lambda x: x.name)]
    assert sel(node_selector={"pool": "h100"}) == [n for n in range(12) if lab[n]["pool"] == "h100"]
    assert sel(node_selector={"pool": "h100", "zone": "b"}) == [n for n in range(12) if lab[n]["pool"] == "h100" and
                                                               lab[n]["zone"] == "b"]

    def term(*exprs):
        return [{"matchExpressions": [dict(key=k, operator=o, values=v) for k, o, v in exprs]}]

    assert sel(node_affinity=term(("pool", "In", ["a100", "cpu"]))) == [n for n in range(12) if lab[n]["pool"] != "h100"]
    assert sel(node_affinity=term(("pool", "NotIn", ["cpu"]), ("zone", "In", ["a"]))) == \
        [n for n in range(12) if lab[n]["pool"] != "cpu" and lab[n]["zone"] == "a"]
    assert sel(node_affinity=term(("gen", "Exists", []))) == [n for n in range(12) if "gen" in lab[n]]
    assert sel(node_affinity=term(("gen", "DoesNotExist", []))) == [n for n in range(12) if "gen" not in lab[n]]
    assert sel(node_affinity=term(("gen", "NotIn", ["8"]))) == [n for n in range(12) if lab[n].get("gen") != "8"]
    # Gt / Lt compare integers; a missing label matches neither
    assert sel(node_affinity=term(("gen", "Gt", ["8"]))) == [n for n in range(12) if int(lab[n].get("gen", "0")) > 8]
    assert sel(node_affinity=term(("gen", "Lt", ["10"]))) == [n for n in range(12) if "gen" in lab[n] and
                                                             int(lab[n]["gen"]) < 10]
    # terms are ORed
    two = term(("pool", "In", ["cpu"])) + term(("gen", "Gt", ["9"]))
    assert sel(node_affinity=two) == [n for n in range(12) if lab[n]["pool"] == "cpu" or
                                      int(lab[n].get("gen", "0")) > 9]


def test_undecidable_selectors():
    _, cls = classes_of(fleet(), keys=("pool",))
    with pytest.raises(NotDecidable):
        role_admit(cls, node_selector={"zone": "a"})
    with pytest.raises(NotDecidable):
        role_admit(cls, node_affinity=[{"matchExpressions": [{"key": "zone", "operator": "Exists"}]}])
    with pytest.raises(NotDecidable):
        role_admit(cls, node_affinity=[{"matchFields": [{"key": "metadata.name", "operator": "In",
                                                          "values": ["n00"]}]}])


def test_more_than_64_classes_is_an_error():
    nodes = [NodeInfo(name=f"n{i:03d}", labels={"rack": str(i)}) for i in range(65)]
    index = NodeIndex([nd.name for nd in nodes], ["d"])
    assert build_node_classes(nodes[:64], NodeIndex([nd.name for nd in nodes[:64]], ["d"]), ("rack",)).n_classes == 64
    with pytest.raises(ValueError):
        build_node_classes(nodes, index, ("rack",))


def test_gt_lt_parse_integers_as_go_parseint():
    """Gt / Lt read label and value with strconv.ParseInt(s, 10, 64): a sign and decimal digits only."""
    for value, ok in (("12", True), ("+12", True), ("-3", True), ("1_2", False), (" 12", False), ("12 ", False),
                      ("0x1f", False), ("9223372036854775808", False), ("", False)):
        nodes = [NodeInfo(name="n0", labels={"gen": value})]
        _, cls = classes_of(nodes, keys=("gen",))
        mask = role_admit(cls, node_affinity=[{"matchExpressions": [{"key": "gen", "operator": "Gt",
                                                                     "values": ["-10"]}]}])
        assert bool(mask) == ok, value
