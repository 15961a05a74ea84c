"""CPU: the batch-reuse fixtures (tests/reuse_cases.py) can tell a call that read the previous call's leftovers from
one that did not.  On the oracles, the large fixture of every family and the small one disagree on the overlapping
prefix of the placements, on the first dense rows and on the alternates; the growth pair sits either side of DevBuf's
growth rule; the failing blobs fail where the tests expect them to."""
import numpy as np
import pytest

import alternates_oracle as ao
import lw_alternates_oracle as lwa
import reuse_cases as rc
from oracle import placer as oracle_placer
from oracle import wave_loop


@pytest.fixture(scope="module")
def plain():
    return rc.plain_world()


def _differ(a, b):
    k = min(len(a), len(b))
    assert k > 0
    return not np.array_equal(np.asarray(a)[:k], np.asarray(b)[:k])


def test_steps_fixtures_differ(plain):
    big = oracle_placer.place(plain.topo, plain.fx[("steps", "large")].blob, want_matrix=True, want_topk=True)
    few = oracle_placer.place(plain.topo, plain.fx[("steps", "small")].blob, want_matrix=True, want_topk=True)
    assert big["rc"] == 0 and few["rc"] == 0
    assert _differ(big["assign"], few["assign"])
    assert not np.array_equal(big["matrix"][0].view(np.uint32), few["matrix"][0].view(np.uint32))
    assert not np.array_equal(big["topk"][0], few["topk"][0])


@pytest.mark.parametrize("wname", ["plain", "levels"])
def test_groups_fixtures_differ(wname, plain):
    w = plain if wname == "plain" else rc.level_world()
    exp = {}
    for size in rc.SIZES:
        groups = wave_loop.groups_from_blob(w.fx[("groups", size)].blob)
        exp[size] = ao.run_fleet_ranked(w.topo, groups, rc.N_ALT)   # (assign, status, domain, score, alt, alt_score)
    assert _differ(exp["large"][0], exp["small"][0])
    assert _differ(exp["large"][3].view(np.uint32), exp["small"][3].view(np.uint32))   # the scores at the picks
    assert _differ(exp["large"][4], exp["small"][4]) and (exp["small"][4] >= 0).any()
    # the first dense rows: the oracle's wave loop, the rows of its first wave (role rows in plan order)
    first = {}
    for size in rc.SIZES:
        waves = []
        wave_loop.run_fleet(w.topo, wave_loop.groups_from_blob(w.fx[("groups", size)].blob), want_matrix=True,
                            want_topk=False, on_wave=lambda wv, act, blob, r: waves.append(r["matrix"]))
        first[size] = waves[0].view(np.uint32)
    k = min(len(first["large"]), len(first["small"]))
    assert all(not np.array_equal(first["large"][i], first["small"][i]) for i in range(k)), k
    # not a prefix: the small fixture's groups are other groups of the fleet, in another order
    assert [g.gid for g in w.fx[("groups", "small")].groups] != [g.gid for g in w.fx[("groups", "large")].groups][:3]


def test_lw_fixtures_differ(plain):
    exp = {s: lwa.run_lw_ranked(plain.topo, plain.fx[("lw", s)].blob, plain.fx[("lw", s)].rp, rc.N_ALT)
           for s in rc.SIZES}
    assert _differ(exp["large"][0], exp["small"][0])
    assert _differ(exp["large"][4], exp["small"][4])
    # the first dense rows: every role row of the first group's first wave
    rows = {s: lwa.run_lw_rows(plain.topo, plain.fx[("lw", s)].blob, plain.fx[("lw", s)].rp)[-1] for s in rc.SIZES}
    firsts = {s: [r.view(np.uint32) for key, r in sorted(rows[s].items()) if key[:2] == min(rows[s])[:2]]
              for s in rc.SIZES}
    assert firsts["small"] and all(not np.array_equal(x, y) for x, y in zip(firsts["large"], firsts["small"]))
    pods = {s: plain.fx[("lw", s)].rp[:, 0] for s in rc.SIZES}
    assert pods["small"].max() < pods["large"].max()   # fewer pods per replica


def test_fixtures_differ_in_shape(plain):
    """Groups, waves, replicas and exclusive groups: the large fixtures have more of each and 8-role waves."""
    import groups_gen as gg
    from rbg_b200.blob import STEP_EXCLUSIVE
    for fam in ("groups", "lw"):
        small, large = (plain.fx[(fam, s)] for s in rc.SIZES)
        assert int(large.blob[2]) > int(small.blob[2]) and int(large.blob[4]) > int(small.blob[4])
        ex = [sum(bool(g.flags & STEP_EXCLUSIVE) for g in f.groups) for f in (small, large)]
        assert ex[1] > ex[0]
    widest = max(len(w) for g in plain.fx[("groups", "large")].groups for w in gg.waves_of(g.roles))
    assert widest == 8
    assert int(plain.fx[("steps", "large")].blob[5]) > int(plain.fx[("steps", "small")].blob[5])


def test_growth_pair_straddles_the_rule(plain):
    a, fits, grows = rc.growth_steps(plain)
    stride = rc.slab_stride(plain.topo.n)
    assert int(a[5]) == 8 and int(fits[5]) == 10 and int(grows[5]) == 11
    cap = rc.grow(8 * stride)
    assert int(fits[5]) * stride <= cap < int(grows[5]) * stride
    ra = oracle_placer.place(plain.topo, a, want_matrix=True, want_topk=False)
    rf = oracle_placer.place(plain.topo, fits, want_matrix=True, want_topk=False)
    assert not np.array_equal(ra["matrix"][0].view(np.uint32), rf["matrix"][0].view(np.uint32))


def test_bad_word_is_the_last_record(plain):
    """The corrupted word is the blob's last one, and host validation (rbgtopo_plan_describe) refuses the blob."""
    from rbg_b200.engine import plan_steps
    gb = plain.fx[("groups", "large")].blob
    bad = rc.bad_word(gb)
    assert np.array_equal(bad[:-1], gb[:-1]) and bad[-1] == -5 and gb[-1] >= 0
    plan_steps(gb, plain.topo.n, len(plain.topo.domain_owner))
    with pytest.raises(RuntimeError, match="-1"):
        plan_steps(bad, plain.topo.n, len(plain.topo.domain_owner))


def test_failing_names_are_the_failing_calls(plain):
    """The GPU module parametrizes its failed-call cases by these names without building the worlds."""
    assert tuple(x[0] for x in rc.failing(plain)) == rc.FAILING_NAMES
    assert tuple(x[0] for x in rc.failing_levels(rc.level0_world())) == rc.ELIMIT_NAMES


def test_level_fixtures_reach_levels():
    w = rc.level_world()
    assert w.flags == dict(lw_committed_levels=True)
    for size in rc.SIZES:
        assert any(g.level > 0 for g in w.fx[("groups", size)].groups)
    z = rc.level0_world()
    assert z.flags == {} and all(g.level == 0 for g in z.fx[("groups", "large")].groups)
    assert np.array_equal(z.lv, w.lv)
