"""CPU: the seeded GROUPS-blob generator of the limit tests (tests/groups_gen.py) reaches what it claims to reach.
Its seed set must cover every limit in groups_gen.BULLETS (status 1 and 2 as the oracle's wave loop computes them),
its wave rule must be the oracle's, and every group must stay under the conservative exactness bound — so an edit
of the generator cannot quietly shrink what tests/test_gpu_groups_limits.py exercises."""
import groups_gen as gg
from oracle import wave_loop


def test_generated_cases_cover_the_abi_limits():
    covered = dict.fromkeys(gg.BULLETS, False)
    for seed, n, scarce, excl in gg.CASES:
        case = gg.make_case(seed, n, scarce=scarce, exclusive=excl)
        states, _ = wave_loop.run_fleet(case.topo, wave_loop.groups_from_blob(case.blob))
        for g, st in zip(case.groups, states):
            assert gg.exact_ok(g, case.wsum_max), (seed, g.gid)
            assert [list(w) for w in st.waves] == gg.waves_of(g.roles), (seed, g.gid)
        for k, v in gg.coverage(case, [st.result()["status"] for st in states]).items():
            covered[k] |= v
    assert all(covered.values()), [k for k, v in covered.items() if not v]


def test_generator_is_deterministic():
    a, b = gg.make_case(4, 130, scarce=True), gg.make_case(4, 130, scarce=True)
    assert (a.blob == b.blob).all() and (a.topo.domain_owner == b.topo.domain_owner).all() and (a.topo.free == b.topo.free).all()
