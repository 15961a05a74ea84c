"""CPU checks of the exclusive-level oracle (DESIGN.md §3.9) and of the host code that accepts the level words."""
import ctypes as C

import numpy as np
import pytest

import levels_oracle as lo
from rbg_b200 import _lib, synth
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE, Group, GroupsBuilder
from rbg_b200.engine import plan_steps


@pytest.mark.parametrize("seed", range(12))
def test_derivation_equals_the_pod_by_pod_terms(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 40))
    n_levels = int(rng.integers(0, 8))
    domain = rng.integers(0, max(1, n // 4) + 1, n).astype(np.int32)
    levels = lo.random_levels(rng, n, domain, n_levels, [bool(rng.random() < 0.5) for _ in range(n_levels)])
    gids = [3, 5, 8, 13][: int(rng.integers(1, 5))]
    occ = lo.random_occ(rng, n, n_levels, gids, int(rng.integers(0, 3 * n + 1)))
    got = lo.derive_level_owner(levels, occ)
    assert np.array_equal(got, lo.owner_from_sets(levels, occ))


@pytest.mark.parametrize("seed", range(8))
def test_derivation_equals_the_reference_terms(seed):
    """The pinned reference terms, evaluated pod by pod with label-selector semantics on both sides, decide for every
    group, level and node exactly what the derived owner vector says."""
    rng = np.random.default_rng(50 + seed)
    n = int(rng.integers(1, 24))
    n_levels = int(rng.integers(0, 4))
    domain = rng.integers(0, max(1, n // 4) + 1, n).astype(np.int32)
    levels = lo.random_levels(rng, n, domain, n_levels, [bool(rng.random() < 0.5) for _ in range(n_levels)])
    gids = [3, 5, 8][: int(rng.integers(1, 4))]
    occ = lo.random_occ(rng, n, n_levels, gids, int(rng.integers(0, 2 * n + 1)))
    assert np.array_equal(lo.derive_level_owner(levels, occ), lo.owner_from_terms(levels, occ, gids + [99]))


def test_seeded_fleets_reach_every_case():
    """The seeds above cover blocked nodes, single owners and free nodes at some level above 0."""
    seen = set()
    for seed in range(12):
        rng = np.random.default_rng(seed)
        n = int(rng.integers(1, 40))
        n_levels = int(rng.integers(0, 8))
        domain = rng.integers(0, max(1, n // 4) + 1, n).astype(np.int32)
        levels = lo.random_levels(rng, n, domain, n_levels, [bool(rng.random() < 0.5) for _ in range(n_levels)])
        gids = [3, 5, 8, 13][: int(rng.integers(1, 5))]
        occ = lo.random_occ(rng, n, n_levels, gids, int(rng.integers(0, 3 * n + 1)))
        own = lo.derive_level_owner(levels, occ)
        seen |= {("blocked" if v == -2 else "free" if v == -1 else "owned") for v in own[1:].ravel()}
    assert seen == {"blocked", "free", "owned"}


# Hand-built cluster: 2 zones (level 0) x 2 NVLink domains x 2 hosts each; level 1 = hostname, level 2 = NVLink domain.
ZONE = np.array([0, 0, 0, 0, 1, 1, 1, 1], dtype=np.int32)
HOST = np.arange(8, dtype=np.int32)
NVL = np.array([0, 0, 1, 1, 2, 2, 3, 3], dtype=np.int32)
LV = np.stack([ZONE, HOST, NVL])
HOSTNAME, ZONE_L = 1, 0


def usable(occ, gid, level, node):
    own = lo.derive_level_owner(LV, occ)[level, node]
    return own in (-1, gid)


def test_two_hostname_groups_share_a_zone_and_an_nvlink_domain_not_a_node():
    occ = [(0, 7, HOSTNAME)]                       # group 7 holds host 0 (hostname key)
    assert usable(occ, 9, HOSTNAME, 1)             # same NVLink domain and zone, other host
    assert usable(occ, 9, HOSTNAME, 3)
    assert not usable(occ, 9, HOSTNAME, 0)         # the node itself
    assert usable(occ, 7, HOSTNAME, 0)


def test_hostname_group_may_not_enter_the_zone_of_a_zone_group():
    occ = [(5, 4, ZONE_L)]                         # group 4 (zone key) holds a pod in zone 1
    for node in range(4, 8):
        assert not usable(occ, 9, HOSTNAME, node)
    for node in range(4):
        assert usable(occ, 9, HOSTNAME, node)


def test_zone_group_may_not_enter_a_zone_that_holds_a_hostname_pod():
    occ = [(2, 7, HOSTNAME)]                       # a hostname-exclusive pod in zone 0
    for node in range(4):
        assert not usable(occ, 4, ZONE_L, node)
    for node in range(4, 8):
        assert usable(occ, 4, ZONE_L, node)


def test_two_groups_in_one_domain_block_everyone():
    occ = [(0, 7, ZONE_L), (1, 8, ZONE_L)]
    own = lo.derive_level_owner(LV, occ)
    assert (own[0, :4] == -2).all() and (own[0, 4:] == -1).all()


@pytest.mark.parametrize("seed", range(6))
def test_level0_records_give_the_legacy_owner_map(seed):
    rng = np.random.default_rng(100 + seed)
    n = int(rng.integers(1, 60))
    n_dom = int(rng.integers(1, 9))
    domain = rng.integers(0, n_dom, n).astype(np.int32)
    occ = np.array([(int(rng.integers(0, n)), int(rng.choice([2, 6])), 0) for _ in range(int(rng.integers(0, 6)))],
                   dtype=np.int32).reshape(-1, 3)
    own = lo.derive_level_owner(domain[None, :], occ)[0]
    assert np.array_equal(own, lo.legacy_owner_map(domain, n_dom, occ)[domain])


def test_group_view_keeps_feasibility_and_numbering():
    topo = synth.make_topology(64, seed=3, tiers=2, owned_frac=0.0, max_free=4)
    rng = np.random.default_rng(3)
    owner0 = rng.choice([-1, -1, -2, 11, 12], size=64).astype(np.int32)
    v = lo.group_view(topo, owner0, 11, 12)
    feasible = v.domain_owner[v.domain]
    assert np.array_equal(feasible == -1, (owner0 == -1) | (owner0 == 11))
    assert np.array_equal(v.domain // 2, topo.domain)


def _one_group(level, fixed=-1, n_dom=4):
    g = Group(gid=5, roles=[(0, 2, 1, ROLE_EXCLUSIVE)], pair=[[1]], flags=STEP_EXCLUSIVE, fixed_domain=fixed,
              level=level)
    return GroupsBuilder().add(g).build()


def test_builder_writes_the_level_words():
    from rbg_b200.blob import BlobBuilder, Step
    gb = _one_group(3)
    assert int(gb[8 + 10]) == 3
    sb = BlobBuilder().add(Step(gid=1, roles=[(1, 1, 0, 0)], level=2)).build()
    assert int(sb[8 + 14]) == 2
    assert int(_one_group(0)[8 + 10]) == 0


def test_describe_calls_accept_the_level_word():
    """The describe calls cannot know level sizes: they accept any level >= 0, range-check fixed_domain at level 0
    only, and the geometry does not change with the level."""
    lib = _lib.load()
    base = plan_steps(_one_group(0), 16, 4)
    assert np.array_equal(plan_steps(_one_group(5), 16, 4), base)
    assert np.array_equal(plan_steps(_one_group(5, fixed=40), 16, 4), base)   # level 5 may have 41+ domains

    def place_rc(gb):
        geom = np.zeros(8, dtype=np.int32)
        order = np.zeros(4, dtype=np.int32)
        gb = np.ascontiguousarray(gb, dtype=np.int32)
        return lib.rbgtopo_place_describe(gb.ctypes.data_as(_lib.i32p), len(gb), 16, 4, None, 0,
                                          order.ctypes.data_as(_lib.i32p), 4, geom.ctypes.data_as(_lib.i32p)), geom

    rc0, g0 = place_rc(_one_group(0))
    rc5, g5 = place_rc(_one_group(5, fixed=40))
    assert rc0 == 0 and rc5 == 0 and np.array_equal(g0, g5)
    assert place_rc(_one_group(0, fixed=40))[0] == -1       # level 0: fixed_domain outside its 4 domains
    assert place_rc(_one_group(-1))[0] == -1
