"""CPU: Node labels -> exclusive-level partitions and pod records (rbg_b200/ingest.py, DESIGN.md §3.9)."""
import random

import numpy as np
import pytest

import levels_oracle as lo
from rbg_b200.ingest import (DEFAULT_TIER_LABELS, NodeInfo, build_exclusive_levels, build_topology,
                             exclusive_occupancy)

NV, HOST, LEAF, ZONE = DEFAULT_TIER_LABELS
HOSTNAME = "kubernetes.io/hostname"
KEYS = (NV, HOSTNAME, ZONE)


def cluster():
    nodes = []
    for i in range(24):
        labels = {NV: f"nvl-{i // 8}", HOSTNAME: f"node-{i:04d}", ZONE: f"z-{i // 12}"}
        if i == 5:
            del labels[ZONE]                       # no zone label: a domain of its own
        nodes.append(NodeInfo(f"node-{i:04d}", labels, {"nvidia.com/gpu": 8}))
    return nodes


def test_partitions_are_deterministic_under_informer_reordering():
    nodes = cluster()
    topo, index = build_topology(nodes)
    lv = build_exclusive_levels(nodes, index, KEYS)
    for seed in range(5):
        shuffled = nodes[:]
        random.Random(seed).shuffle(shuffled)
        t2, i2 = build_topology(shuffled)
        lv2 = build_exclusive_levels(shuffled, i2, KEYS)
        assert np.array_equal(lv.domain, lv2.domain) and np.array_equal(lv.n_domains, lv2.n_domains)
    assert lv.domain.shape == (2, 24)
    assert list(lv.n_domains) == [24, 3]            # 24 hosts; 2 zones + the unlabelled node
    assert len(set(lv.domain[1][[0, 1, 2, 3, 4, 6]])) == 1 and lv.domain[1][5] not in lv.domain[1][[0, 12]]


def test_records_name_the_level_of_the_groups_key():
    nodes = cluster()
    topo, index = build_topology(nodes)
    lv = build_exclusive_levels(nodes, index, KEYS)
    pods = [("node-0003", 7, HOSTNAME), ("node-0013", 4, ZONE), ("gone", 9, ZONE), ("node-0001", 8, NV)]
    occ = exclusive_occupancy(lv, index, pods)
    assert occ.tolist() == sorted([[index.node_id("node-0003"), 7, 1], [index.node_id("node-0013"), 4, 2],
                                   [index.node_id("node-0001"), 8, 0]])
    with pytest.raises(ValueError):
        exclusive_occupancy(lv, index, [("node-0001", 3, "unknown/key")])
    own = lo.derive_level_owner(np.vstack([topo.domain[None, :], lv.domain]), occ)
    # the zone-keyed pod of group 4 blocks zone 1 for everyone else at every level ...
    z1 = [index.node_id(f"node-{i:04d}") for i in range(12, 24)]
    assert (own[1][z1] != -1).all()
    # ... the hostname pod of group 7 takes its own host; the NVLink-keyed pod of group 8 takes nvl-0 from everyone,
    # so host 3 (in nvl-0) is blocked for all, and a host of nvl-1 in zone 0 stays free at the hostname level
    assert own[1][index.node_id("node-0003")] == -2
    assert own[1][index.node_id("node-0002")] == 8
    assert own[1][index.node_id("node-0009")] == -1
