"""CPU: the fleets of tests/wide_matrix_cases.py still reach the 2^31-element edge of the dense matrix (every `*_pre`
check at full size), and the premise that lets the GPU tests run the oracle once per distinct group holds: at a
scaled-down N, the oracle of the whole fleet equals the oracle of each distinct group alone, copied to every group it
stands for."""
import numpy as np
import pytest

import wide_matrix_cases as wm


@pytest.fixture(scope="module")
def fleet():
    return wm.groups_fleet()


@pytest.fixture(scope="module")
def groups_ref(fleet):
    return wm.groups_oracle(fleet, subset=[0] + list(wm.STRADDLE))


def test_layout():
    wm.layout_pre()


def test_groups_fleet_reaches_the_straddle(fleet, groups_ref):
    at = wm.plan_pre(fleet)
    assert {g for _, _, g, _ in at.values()} == {890, 891}
    wm.anchors_pre(fleet)
    _, rows, _ = groups_ref
    rows_of = lambda g: rows[(fleet.rep[g], 0)]
    wm.wrap_alias_pre(rows_of)
    wm.best_above_pre(rows_of, fleet)


def test_steps_fleet_reaches_the_straddle():
    sf = wm.steps_fleet()
    wm.steps_pre(sf)
    ref = wm.steps_oracle(sf, subset=[0] + sf.hub_steps)
    for c in wm.CHUNKS:                       # the straddling step's rows: defined and not constant past n*
        r, nstar = wm.straddle(wm.N, c)
        row = ref[r // wm.Q]["matrix"][r % wm.Q]
        assert np.isfinite(row[nstar:]).sum() > 1000 and len(np.unique(row[nstar:])) > 10, c
        assert (ref[0]["matrix"][0][:wm.N - nstar].view(np.uint32) != row[nstar:].view(np.uint32)).any(), c


def test_rerun_fleet_is_rerun(fleet):
    rf = wm.rerun_fleet(topo=fleet.topo)
    per, rows, _ = wm.groups_oracle(rf)
    wm.rerun_pre(rf, lambda g: int(per[g][1][0]))
    assert all((g, 1) in rows for g in rf.distinct)          # the second wave of every group runs


SMALL_N, SMALL_G = 4096, 14
SMALL_STRADDLE = (6, 7, 8, 9)


def _same(x, y, tag):
    x, y = np.asarray(x), np.asarray(y)
    if x.dtype.kind == "f":
        x, y = x.view(np.uint32), y.view(np.uint32)
    assert x.shape == y.shape and np.array_equal(x, y), tag


def test_whole_groups_fleet_equals_distinct_groups():
    from oracle import wave_loop
    import alternates_oracle
    f = wm.groups_fleet(SMALL_N, SMALL_G, SMALL_STRADDLE)
    per, rows, topk = wm.groups_oracle(f)
    waves = []
    wave_loop.run_fleet(f.topo, wave_loop.groups_from_blob(f.blob), want_matrix=True, want_topk=True,
                        on_wave=lambda w, act, blob, r: waves.append(r))
    assert len(waves) == 1
    whole = waves[0]
    for g in range(SMALL_G):
        _same(whole["matrix"][wm.Q * g:wm.Q * (g + 1)], rows[(f.rep[g], 0)], ("rows", g))
        _same(whole["topk"][wm.Q * g:wm.Q * (g + 1)], topk[(f.rep[g], 0)], ("topk", g))
    exp = wm.expand(f, per, wm.replica_spans(f))
    got = alternates_oracle.run_fleet_ranked(f.topo, wave_loop.groups_from_blob(f.blob), 8)
    for name, x in zip(("assign", "status", "domain", "score", "alt_node", "alt_score"), got):
        _same(x, getattr(exp, name), name)


def test_whole_rerun_fleet_equals_distinct_groups():
    from oracle import wave_loop
    import alternates_oracle
    f = wm.rerun_fleet(SMALL_N, SMALL_G, SMALL_STRADDLE)
    per, _, _ = wm.groups_oracle(f)
    exp = wm.expand(f, per, wm.replica_spans(f))
    got = alternates_oracle.run_fleet_ranked(f.topo, wave_loop.groups_from_blob(f.blob), 8)
    assert (got[1] == 1).all()
    for name, x in zip(("assign", "status", "domain", "score", "alt_node", "alt_score"), got):
        _same(x, getattr(exp, name), name)


def test_whole_lw_fleet_equals_distinct_groups():
    f = wm.groups_fleet(SMALL_N, SMALL_G, SMALL_STRADDLE)
    rp = wm.lw_role_pods(f)
    assert {tuple(x) for x in rp} >= {(s, c) for s in (1, 2, 4) for c in (-1, 0, 1)}
    spans = wm.lw_spans(f, rp)
    per = wm.lw_oracle(f, rp)
    exp = wm.expand(f, per, spans)
    whole = wm.lw_oracle(f, rp, subset=range(SMALL_G))
    for g in range(SMALL_G):
        for k, name in enumerate(("assign", "status", "domain", "score", "alt_node", "alt_score")):
            want = getattr(exp, name)[g] if k in (1, 2) else getattr(exp, name)[spans[g]]
            _same(whole[g][k], want, (name, g))


def test_whole_steps_fleet_equals_distinct_steps():
    from oracle import placer as oracle_placer
    f = wm.steps_fleet(SMALL_N, SMALL_G, SMALL_STRADDLE)
    per = wm.steps_oracle(f)
    whole = oracle_placer.place(f.topo, f.blob, want_matrix=True, want_topk=True)
    assert whole["rc"] == 0
    for s in range(SMALL_G):
        r, sl = per[f.rep[s]], slice(wm.Q * s, wm.Q * (s + 1))
        for name in ("assign", "matrix", "topk"):
            _same(whole[name][sl], r[name], (name, s))
        assert (whole["status"][s], whole["domain"][s]) == (r["status"][0], r["domain"][0]), s
