"""CPU: the committed-batch generator (tests/commit_gen.py) reaches every bullet it lists with the seed set of the GPU
tests, and every group it makes is under the exactness bound."""
import groups_gen as gg
import commit_gen as cg
from committed_oracle import run_fleet_committed, run_fleet_snapshot
from oracle import wave_loop


def test_seed_set_reaches_every_bullet_and_every_group_is_exact():
    cs = cg.cases()
    results = {}
    for case in cs:
        assert all(gg.exact_ok(g, gg.wsum_max(case.topo)) for g in case.groups), case.name
        groups = wave_loop.groups_from_blob(case.blob)
        results[case.name] = (run_fleet_committed(case.topo, groups, fast=True),
                              run_fleet_snapshot(case.topo, groups))
    cov = cg.coverage(cs, results)
    assert all(cov.values()), [k for k, v in cov.items() if not v]


def test_chains_fill_one_node_per_group():
    """The oracle's side of the chain: group i takes the i-th node of the background order, nobody fails."""
    case = cg.chain(16, 16, 2)
    states = run_fleet_committed(case.topo, wave_loop.groups_from_blob(case.blob), fast=True)
    nodes = [s.assign_in_group_order()[0] for s in states]
    assert sorted(nodes) == list(range(16)) and all(s.result()["status"] == 0 for s in states)


def test_hub_fills_exactly():
    case = cg.hub()
    states = run_fleet_committed(case.topo, wave_loop.groups_from_blob(case.blob), fast=True)
    used = sum(g.roles[0][2] * sum(1 for x in s.assign_in_group_order() if x == 0) for g, s in zip(case.groups, states))
    assert used == cg.HUB_FREE
    st = [s.result()["status"] for s in states]
    assert st[-4:] == [0, 1, 2, 0] and all(x == 0 for x in st[:-3])


def test_two_reporters_depend_on_the_last_one():
    """The gid-11 group after two reporters of D (gids 11, then 12) stays out of D; were D owned by the first
    reporter, it would take D's best node."""
    import copy
    from committed_oracle import run_group
    for case in (cg.two_reporters(0), cg.two_reporters(1)):
        groups = wave_loop.groups_from_blob(case.blob)
        d = case.groups[0].fixed_domain
        states = run_fleet_committed(case.topo, groups)
        assert [s.result()["domain"] for s in states[:2]] == [d, d] and states[2].result()["domain"] != d
        first_wins = copy.copy(case.topo)
        first_wins.domain_owner = case.topo.domain_owner.copy()
        first_wins.domain_owner[d] = 11
        claimed = {}
        for s in states[:2]:
            for x in s.assign_in_group_order():
                if x >= 0:
                    claimed[x] = claimed.get(x, 0) + 1
        assert run_group(first_wins, groups[2], claimed).result()["domain"] == d
