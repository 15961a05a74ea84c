"""CPU: the preconditions of tests/commit_levels_limits_cases.py, asserted on the committed-levels oracle alone
(committed_levels_oracle.run_fleet_committed_levels and its `terms` / `reporter` switches), and the seed set's
coverage."""
import numpy as np
import pytest

import commit_gen as cg
import commit_levels_limits_cases as cl
from oracle import wave_loop
from rbg_b200.blob import STEP_EXCLUSIVE

CHAIN_IDS = [f"{k}{G}" for G, k in cl.CHAINS]


@pytest.mark.parametrize("G,kind", cl.CHAINS, ids=CHAIN_IDS)
def test_chains_take_exactly_G_rounds_through_their_term(G, kind):
    c = cl.chain(G, kind)
    f = cl.chain_facts(c)
    assert f["alternates"] and f["all_placed"], f
    assert f["rounds"] == G == c.rounds and f["replay_final"] and f["settles_in_round_i"], f
    if kind == "P":
        assert f["without_P"] and not f["without_K"], f
    elif kind == "K":
        assert f["without_K"] and not f["without_P"], f
        assert f["lmask"] == (1 << 3 | 1 << 6)               # neither contiguous nor holding level 0
    else:
        assert f["without_K"] and f["lmask"] == 0xFF, f


def test_refresh_chain_alternates_at_every_level():
    c = cl.chain(*cl.REFRESH_CHAIN)
    f = cl.chain_facts(c, replay=False)
    assert f["alternates"] and f["all_placed"] and f["lmask"] == 0xFF, f


@pytest.mark.parametrize("i", range(len(cl.SPARSE) * 2))
def test_sparse_masks(i):
    c = cl.sparse_cases()[i]
    ex, others = cl.SPARSE[i // 2]
    assert cl.lmask(c.blob) == sum(1 << L for L in ex)
    gr = c.extra["groups"]
    outside = {g.level for g in gr if not g.flags & STEP_EXCLUSIVE and cg.pending(g) > 0}
    assert outside and outside <= set(others) and min(outside) >= 1 and cl.uses_levels(c.blob)
    assert all(g.fixed_domain < c.nd[g.level] for g in gr)
    a, s, d = cl.expected(c)
    assert (s == 0).any()


def test_level_offset_edges_claim_both_boundary_ids():
    c = cl.offsets()
    f = cl.offsets_facts(c)
    assert f["claimed_all"] and f["levels"] == 8 and f["idle"] == 6 and f["readers"] == 14, f
    assert sum(f["moved"]) >= 7, f
    assert not np.array_equal(cl.expected(c, terms=("P",))[0], cl.expected(c)[0])


def test_long_pod_list_in_one_zone():
    c = cl.pods()
    assert c.topo.n <= 10_000
    f = cl.pods_facts(c)
    assert f["max_pods"] >= 2000 and f["without_P"] and f["zone_readers_out"][0] == 1, f


def test_gid_edges():
    f = cl.gids_facts(cl.gids())
    assert all(f[k] for k in ("gid_ends", "shared_gid_matters", "reporters", "last_reporter_keeps_out",
                              "first_differs", "blocked")), f
    assert f["same_gid_levels"] == [1, 6]


@pytest.mark.parametrize("i", range(len(cl.level0_pairs())))
def test_moved_non_exclusive_groups_keep_the_level0_results(i):
    base, moved = cl.level0_pairs()[i]
    assert not cl.uses_levels(base.blob) and cl.uses_levels(moved.blob) and cl.lmask(moved.blob) in (0, 1)
    for g in moved.extra["groups"]:
        assert g.fixed_domain < moved.nd[g.level]
    for x, y in zip(cl.expected(base), cl.expected(moved)):
        assert np.array_equal(x, y)


def test_literal_and_replayed_oracles_agree():
    """The replay of the rounds (place_one) ends on the sequential oracle's results on generated batches."""
    for c in cl.sparse_cases()[:2] + [cl.offsets()]:
        rounds, hist = cl.replay_rounds(c)
        assert [cl._key(s) for s in hist[-1]] == [cl._key(s) for s in cl.states(c)]
        assert 1 <= rounds <= int(c.blob[2])


def test_coverage():
    cs = cl.cases()
    snap, comm = {}, {}
    for c in cs:
        if c.name.startswith("chain"):
            continue
        groups = wave_loop.groups_from_blob(c.blob)
        own = cl.owner(c)
        res = lambda s: (s.assign_in_group_order(), s.result()["status"], s.result()["domain"])
        snap[c.name] = [res(cl.place_one(c, g, [], groups, own)) for g in range(len(groups))]
        comm[c.name] = [res(s) for s in cl.states(c)]
    cov = cl.coverage(cs, snap, comm)
    assert all(cov.values()), [k for k, v in cov.items() if not v]
