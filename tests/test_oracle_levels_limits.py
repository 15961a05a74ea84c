"""CPU checks of tests/levels_limits_cases.py: every case reaches the limit it exists for (stride counts taken with the
132 SMs of an H100), the vectorised derivation equals the literal one of DESIGN.md §3.9 word for word, and
unused_gid gives an "other" owner that no group uses and that fits int32."""
import numpy as np
import pytest

import levels_limits_cases as C
import levels_oracle as lo
import levels_view as lvw
from rbg_b200.blob import STEP_GANG


def test_derivation_case_passes_every_stride():
    c = C.derivation()
    f = C.derivation_facts(c, lo.derive_level_owner_fast(c.lv, c.occ))
    assert f["n"] == (1 << 20) + 1 and f["levels"] == 7 and f["ragged"]
    assert f["records"] >= 600_000 and f["records"] > 2 * C.H100_SMS * 8 * 256
    assert f["phase0"] >= 2 and f["phase1"] >= 3 and f["phase2"] >= 2, f
    assert f["contention_records"] >= 100_000 and f["contention_gids"] >= 3000
    assert f["same_gid_records"] == 50_000 and f["gids_at_ends"] and f["keyed7_only_at_7"] and f["crowd_gids"] == 32
    for k in ("contention_blocked", "same_gid_kept", "ends_kept", "keyed7_everywhere", "crowd_blocked"):
        assert f[k], k
    assert f["kinds"] == {-2, -1, 0}
    # level 3 (racks of 256 offset by 128) does not nest in level 0 (4 096-node domains)
    pairs = np.unique(c.lv[3].astype(np.int64) << 32 | c.lv[0])
    assert len(pairs) > len(np.unique(c.lv[3]))


@pytest.mark.parametrize("n", [1, 33, 4097])
def test_fast_derivation_equals_the_literal_one(n):
    """The derivation case's shapes (hostname, racks, a non-nesting level, one domain, sparse declared counts, gids 0
    and 2^31 - 1) at a size the literal oracle takes."""
    rng = np.random.default_rng(n)
    ids = np.arange(n)
    lv = np.stack([ids // 16, ids, ids // 4, (ids + 2) // 8, np.zeros(n, np.int64), rng.permutation(n), 2 * ids,
                   rng.integers(0, 2 * n, n)]).astype(np.int32)
    occ = np.concatenate([
        np.stack([rng.integers(0, n, 3 * n), rng.integers(0, 6, 3 * n), rng.choice([0, 1, 2, 3, 5, 6, 7], 3 * n)], 1),
        [[0, 0, 7], [n - 1, C.GID_MAX, 1], [n // 2, C.GID_MAX, 4]]]).astype(np.int32)
    assert np.array_equal(lo.derive_level_owner_fast(lv, occ), lo.derive_level_owner(lv, occ))
    assert np.array_equal(lo.derive_level_owner_fast(lv, occ[:0]), lo.derive_level_owner(lv, occ[:0]))


def test_fast_derivation_equals_the_literal_one_on_the_case_builders():
    """Every derivation case of the module: the million-node ones (derivation, hostname_1m) by the same builders at a
    reduced N, the others at full size."""
    cases = [C.keys47(*a) for a in C.KEYS47] + [C.ragged(n) for n in C.RAGGED] + [C.gid_ends(), C.wide47()]
    cases += [C.derivation(n=4097), C.derivation(n=8193, seed=2), C.level_split()]
    topo, seq = C.reinstalls(n=513)
    rows = None
    for lvl, occ, _ in seq:
        rows = lvl if lvl is not None else rows
        cases.append(C.LevelsCase(topo, np.vstack([topo.domain[None], rows]), [], occ))
    h = C.hostname_1m(n=2049)
    cases.append(h)
    cases.append(C.ceiling())
    for c in cases:
        assert np.array_equal(lo.derive_level_owner_fast(c.lv, c.occ), lo.derive_level_owner(c.lv, c.occ))
    assert C.hostname_facts(h, lo.derive_level_owner_fast(h.lv, h.occ))["only_usable_7"]


def test_fast_derivation_under_contention_at_full_size():
    """Thousands of gids on one domain and tens of thousands of records of one gid on one node: the literal oracle over
    a few nodes (the records loop is what it does per record) against the fast one."""
    rng = np.random.default_rng(9)
    n = 64
    ids = np.arange(n)
    lv = np.stack([ids // 16, ids, ids // 4, np.zeros(n, np.int64)]).astype(np.int32)
    i = np.arange(100_000)
    occ = np.concatenate([np.stack([i % 16, 10_000 + i % 3000, i % 3], 1),
                          np.stack([np.full(50_000, 40), np.full(50_000, 7), np.arange(50_000) % 3], 1),
                          np.stack([rng.integers(48, 64, 200), rng.integers(0, 3, 200), np.full(200, 1)], 1)])
    fast = lo.derive_level_owner_fast(lv, occ)
    assert np.array_equal(fast, lo.derive_level_owner(lv, occ))
    assert (fast[:, :16] == lo.BLOCKED).all() and int(fast[1, 40]) == 7


def test_reinstall_sequence_grows_the_tables():
    topo, seq = C.reinstalls()
    totals = [len(topo.domain_owner) + sum(nd) for lvl, _, nd in seq if lvl is not None]
    assert [len(lvl) for lvl, _, _ in seq if lvl is not None] == [7, 2, 7]
    assert totals[2] > totals[0] > totals[1]
    assert all(len(np.unique(r)) == topo.n for r in seq[0][0])          # hostname-like levels
    assert len(seq[3][1]) == 0 and len(seq[4][1]) > 0


def test_keys47_cases_reach_every_corner():
    seen = dict(status1=set(), gang_failed=False, single=False, fixed0=False, last7=False, nonsingle=False)
    for a in C.KEYS47:
        c = C.keys47(*a)
        owner = lo.derive_level_owner_fast(c.lv, c.occ)
        exp, _ = lvw.expected_fleet(c.topo, c.lv, owner, c.nd, c.gblob)
        f = C.keys47_facts(c, exp, owner)
        assert f["levels"] == {4, 5, 6, 7} and f["fixed_in_level"] and f["last_domain_l7"]
        assert f["nested"] and f["non_nested"]
        # owner_L and owner_{L-4} tell some node of a domain a group placed in apart: a 2-bit level read shows
        assert f["split_in_placed_domains"] > 0, a
        seen["status1"] |= set(f["status1_at_47"])
        seen["gang_failed"] |= f["gang_failed"]
        seen["single"] |= f["single_domain"]
        seen["nonsingle"] |= not f["single_domain"]
        seen["fixed0"] |= f["fixed_0_single"]
    assert seen["status1"] == {4, 5, 6, 7} and seen["gang_failed"] and seen["single"] and seen["nonsingle"]
    assert seen["fixed0"]


def test_level_split_case_separates_l_from_l_minus_4():
    """Groups 50 and 52 (level 6) and 51 (level 7) place in domains whose best nodes are free at L and blocked at
    L - 4; group 53 (level 7) is the control whose domain level 3 leaves free."""
    c = C.level_split()
    owner = lo.derive_level_owner_fast(c.lv, c.occ)
    exp, _ = lvw.expected_fleet(c.topo, c.lv, owner, c.nd, c.gblob)
    assert [e[1] for e in exp] == [0, 0, 0, 0]
    gids = [50, 51, 52, 53]
    levels = [6, 7, 6, 7]
    split = [C.split_nodes(c, owner, g, L, e[2]) for g, L, e in zip(gids, levels, exp)]
    assert split[0] == 16 and split[1] == 8 and split[2] == 16 and split[3] == 0, split
    assert exp[0][0] == [16] * 3 and exp[1][0][:4] == [136] * 4 and exp[2][0] == [16] * 2
    # the nodes L - 4 blocks are the best of the domain: free 4 where every other node has 2
    for lo_, hi, L in ((16, 24, 2), (136, 144, 3)):
        assert (c.topo.free[lo_:hi] == 4).all()
        assert (owner[L, lo_:hi] >= 0).all() and (owner[L + 4, lo_:hi] == lo.FREE).all()


def test_hostname_case_at_a_million_nodes():
    h = C.hostname_1m()
    f = C.hostname_facts(h, lo.derive_level_owner_fast(h.lv, h.occ))
    assert f["n"] == (1 << 20) + 1 and f["hostname_5"] and f["hostname_7"] and f["uniform_free"]
    assert f["last_alone"] and f["others_deg"] > 0           # lowest base, highest id: last in the background order
    assert f["only_usable_5"] and f["only_usable_7"]
    gb = h.gblob
    assert bool(gb[8 + 12 * 3 + 1] & STEP_GANG) and not gb[8 + 12 * 2 + 1] & STEP_GANG


def test_derivation_builder_keeps_its_shapes_at_reduced_n():
    """The reduced cases the literal oracle checks above have the records the full-size case exists for."""
    for n in (4097, 8193):
        c = C.derivation(n=n)
        f = C.derivation_facts(c, lo.derive_level_owner_fast(c.lv, c.occ))
        for k in ("contention_blocked", "same_gid_kept", "ends_kept", "keyed7_everywhere", "crowd_blocked"):
            assert f[k], (n, k)
        assert f["gids_at_ends"] and f["keyed7_only_at_7"] and f["crowd_gids"] == 32 and f["kinds"] == {-2, -1, 0}


def test_ceiling_case_sits_on_the_limit():
    assert C.ceiling().total_domains == C.MAX_TOTAL_DOMAINS
    assert C.ceiling(over=1).total_domains == C.MAX_TOTAL_DOMAINS + 1
    assert C.grid_strides(2 * C.MAX_TOTAL_DOMAINS) > 1
    # where a 32-bit index would overflow: the last index below the bound plus one grid stride
    stride = C.H100_SMS * 8 * 256
    assert 2 * C.MAX_TOTAL_DOMAINS - 1 + stride > (1 << 31) - 1


@pytest.mark.parametrize("gids", [[0], [C.GID_MAX], [0, C.GID_MAX], [0, 1, 2, C.GID_MAX], [5, 5, 7],
                                  list(range(100)) + [C.GID_MAX]])
def test_unused_gid_is_unused_and_fits_int32(gids):
    g = lo.unused_gid(gids)
    assert g not in gids and 0 <= g <= C.GID_MAX
    assert g == min(x for x in range(len(gids) + 2) if x not in gids)
