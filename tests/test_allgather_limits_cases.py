"""CPU: the designed cases of tests/allgather_limits_cases.py on the oracles alone.  Every case still reaches its edge
(its `*_pre`), and the numpy shard protocol (per-slab lists, merge, restricted reselect, merge + greedy) at each world the
case names gives the world = 1 oracle's placements, D* and final lists.  For plans, every wave the oracle's wave loop
runs goes through the protocol the same way, and its rows are where the staged plan keeps them."""
import numpy as np
import pytest

import allgather_limits_cases as C
from oracle import placer as oracle_placer
from rbg_b200.engine import plan_steps


@pytest.mark.parametrize("family,name", C.all_step_cases())
def test_step_case(family, name):
    topo, blob, info = C.step_case(family, name)
    ref = C.step_pre(family, name, topo, blob, info)
    for world in info["worlds"] + (2,):
        assign, status, dstar, topk = C.protocol_topk(topo, blob, world, ref)
        assert np.array_equal(assign, ref["assign"]), (world, assign, ref["assign"])
        assert np.array_equal(status, ref["status"]) and np.array_equal(dstar, ref["domain"]), world
        assert np.array_equal(topk, ref["topk"]), world


@pytest.mark.parametrize("name", C.PLAN_CASES)
def test_plan_case(name):
    topo, gblob, info = C.plan_case(name)
    states, waves = C.plan_pre(name, topo, gblob, info)
    first = {(int(st[0]), int(st[1])): int(st[4]) for st in plan_steps(gblob, topo.n, len(topo.domain_owner))}
    for w, gis, blob, r in waves:
        again = oracle_placer.place(topo, blob)
        assert np.array_equal(again["assign"], r["assign"]) and np.array_equal(again["matrix"], r["matrix"])
        for world in info["worlds"]:
            assign, status, dstar, topk = C.protocol_topk(topo, blob, world, r)
            assert np.array_equal(assign, r["assign"]) and np.array_equal(status, r["status"]), (w, world)
            assert np.array_equal(dstar, r["domain"]) and np.array_equal(topk, r["topk"]), (w, world)
        assert all((gi, w) in first for gi in gis)
    # the plan's rows of a group's waves are consecutive, in group order
    rows = sorted(first.items(), key=lambda kv: kv[1])
    assert [k for k, _ in rows] == sorted(first)


def test_peer_bytes_rule():
    topo, gblob, _ = C.plan_case("chain")
    ph = C.phases_rows("plan", gblob, topo)
    assert ph[0][0] == 2 and ph[-1][0] == 1                      # the exclusive group's waves take a second phase
    topo, blob, _ = C.excl_case("far_w3")
    assert C.phases_rows("steps", blob, topo) == [(2, 3)]
    topo, blob, _ = C.merge_case("ksmall_w3")
    assert C.peer_bytes("steps", blob, topo, 3) == 2 * 32 * 8 * 2
