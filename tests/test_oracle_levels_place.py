"""CPU: the level view of levels_view places exclusive groups at their level L as the reference's required terms demand
(DESIGN.md §3.9): over random nested and non-nested partitions and random pod records, no pod the view-based wave loop
places for a participating role breaks a required anti-affinity term against the records, and every such pod lies in
the group's reported level-L domain."""
import numpy as np
import pytest

import groups_gen as gg
import levels_oracle as lo
import levels_view as lvw


@pytest.mark.parametrize("seed", range(8))
def test_level_view_placements_respect_the_terms(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.choice([17, 64, 150]))
    case = gg.make_case(seed, n, scarce=seed % 3 == 0, exclusive=True)
    topo = case.topo
    lv = lo.random_levels(rng, n, topo.domain, 3, [bool(b) for b in rng.integers(0, 2, 3)])
    nd = [len(topo.domain_owner)] + [int(lv[L].max()) + 1 for L in range(1, 4)]
    ng = int(case.blob[2])
    gb = lvw.with_levels(case.blob, [int(rng.integers(0, 4)) for _ in range(ng)])
    for g in range(ng):
        if gb[8 + 12 * g + 2] >= 0:
            gb[8 + 12 * g + 2] = -1
    gids = [int(gb[8 + 12 * g]) for g in range(ng)]
    occ = lo.random_occ(rng, n, 3, gids[:3] + [999], max(1, n // 5))
    owner = lo.derive_level_owner(lv, occ)
    exp, _ = lvw.expected_fleet(topo, lv, owner, nd, gb)
    keys = [f"example.com/level-{L}" for L in range(4)]
    offs = np.concatenate([[0], np.cumsum([int(gb[8 + 12 * g + 9]) for g in range(ng)])]).astype(int)
    for g in range(ng):
        rec = gb[8 + 12 * g: 8 + 12 * g + 12]
        if not rec[1] & 1:
            continue
        L, (assign, _status, dom) = int(rec[10]), exp[g]
        roles = gb[rec[4]: rec[4] + 4 * rec[3]].reshape(-1, 4)
        part = [bool(ro[3] & 1) for ro in roles for _ in range(ro[1])]
        assert len(part) == offs[g + 1] - offs[g] == len(assign)
        for node, p in zip(assign, part):
            if node < 0 or not p:
                continue
            assert not lo.violates(lv, keys, occ, gids[g], L, node), (g, node)
            assert lv[L, node] == dom, (g, node, dom)
