"""CPU: the host-side plan geometry of rbgtopo_place_groups (rbgtopo_plan_describe runs the
very code path, without a device) against the wave planning of the plugin mirror
(rbg_b200/plugin.py::_GroupRun), which the GPU tests in turn check against the oracle."""
import ctypes as C

import numpy as np
import pytest

from rbg_b200 import _lib, synth
from rbg_b200.plugin import (EXCLUSIVE_TOPOLOGY_KEY, GANG_SCHEDULING_KEY, B200TopoPodGroupManager, RoleBasedGroup,
                             RoleSpec, _GroupRun)
from test_plugin_host import OraclePlacer

I32P = C.POINTER(C.c_int32)


def describe(blob, n_nodes=4096, n_domains=64, degp1=None, wsum_max=0):
    lib = _lib.load()
    blob = np.ascontiguousarray(blob, dtype=np.int32)
    cap = 1 << 16
    out = np.zeros(cap * 8, dtype=np.int32)
    ns, nw, pw = C.c_int32(), C.c_int32(), C.c_int64()
    dp = None if degp1 is None else np.ascontiguousarray(degp1, dtype=np.int32).ctypes.data_as(I32P)
    rc = lib.rbgtopo_plan_describe(blob.ctypes.data_as(I32P), len(blob), n_nodes, n_domains, dp, wsum_max,
                                   out.ctypes.data_as(I32P), cap, C.byref(ns), C.byref(nw), C.byref(pw))
    return rc, out[:ns.value * 8].reshape(-1, 8), nw.value, pw.value


def _fleet(n_groups, seed):
    shapes = [synth.shape_mooncake(), synth.shape_pd_144(), synth.shape_fleet8(), synth.shape_sglang_pd()]
    rng = np.random.default_rng(seed)
    out = []
    for g in range(n_groups):
        sh = shapes[g % len(shapes)]
        roles = [RoleSpec(r.name, int(r.replicas), tuple(r.deps), r.demand) for r in sh.roles]
        if g % 5 == 0:
            roles[-1].replicas = int(rng.integers(33, 100))    # several waves of 32
        if g % 7 == 0:
            roles[0].replicas = 0                              # nothing pending in a role
        ann = {}
        if g % 3 == 0:
            ann[EXCLUSIVE_TOPOLOGY_KEY] = "zone"
        if g % 4 == 0:
            ann[GANG_SCHEDULING_KEY] = "true"
        out.append(RoleBasedGroup("default", f"rbg{g}", roles, annotations=ann, gid=g, policy_rules=sh.policy_rules,
                                  placed=[(sh.roles[0].name, int(rng.integers(0, 4096)))] if g % 2 else []))
    return out


@pytest.mark.parametrize("n_groups,seed", [(1, 0), (7, 1), (150, 2)])
def test_plan_geometry_matches_the_plugin_wave_planner(n_groups, seed):
    topo = synth.make_topology(256, seed=1, tiers=2)
    mgr = B200TopoPodGroupManager(OraclePlacer(topo))
    rbgs = _fleet(n_groups, seed)
    blob, _ = mgr.groups_blob(rbgs)
    rc, steps, n_waves, plan_words = describe(blob)
    assert rc == 0
    runs = [_GroupRun(r, mgr.arith) for r in rbgs]
    assert n_waves == max((len(g.waves) for g in runs), default=0)
    # expected: wave-major, groups in order
    exp = []
    for w in range(n_waves):
        for gi, g in enumerate(runs):
            if w < len(g.waves):
                exp.append((gi, w))
    assert [(int(s[0]), int(s[1])) for s in steps] == exp
    row = 0
    off = 8 + 16 * len(steps)
    first_step = {}
    group_off, acc = [], 0          # dense rows / assign indices are in GROUP order (the blob's assign_off)
    for g in runs:
        group_off.append(acc)
        acc += sum(g.pending)
    for i, (s, (gi, w)) in enumerate(zip(steps, exp)):
        g = runs[gi]
        wave = g.waves[w]
        R = sum(c for _, _, c in wave.roles)
        P = len(wave.roles)
        i0 = sum(c for ww in g.waves[:w] for _, _, c in ww.roles)
        na = len(g.anchors)
        assert (int(s[4]), int(s[5]), int(s[7])) == (group_off[gi] + i0, row, i0), (i, gi, w)
        size = (4 * P + P * g.Q + 3 * (na + i0) + 2 * i0 + 3) & ~3
        assert (int(s[2]), int(s[3])) == (off, off + size), (i, gi, w)
        nxt = exp.index((gi, w + 1)) if w + 1 < len(g.waves) else 0
        assert int(s[6]) == nxt
        row += P
        off += size
        first_step.setdefault(gi, i)
    assert plan_words == off


def test_plan_describe_rejects_what_place_groups_rejects():
    topo = synth.make_topology(256, seed=1, tiers=2)
    mgr = B200TopoPodGroupManager(OraclePlacer(topo))
    blob, _ = mgr.groups_blob(_fleet(5, 3))
    bad = blob.copy()
    bad[4] += 1                                   # total pending
    assert describe(bad)[0] == -1
    bad = blob.copy()
    bad[8 + 3] = 99                               # q of group 0
    assert describe(bad)[0] == -6                 # RBGTOPO_ELIMIT
    rc, steps, _, _ = describe(blob, n_nodes=3)   # anchors beyond the node count
    assert rc == -1
    # exactness bound: heavy rows make the scores leave the exact fp32 range
    assert describe(blob, wsum_max=10 ** 7)[0] == -4


@pytest.mark.parametrize("seed,n", [(s, n) for s, n, _, _ in __import__("groups_gen").CASES] + [(20 + s, 512) for s in range(6)])
def test_oracle_wave_split_matches_plan_describe_at_the_abi_limits(seed, n):
    """Generated GROUPS blobs (16-role groups, levels of 9+ pending roles, waves of exactly 8 role rows / 32 replicas,
    zero-pending roles and levels): the oracle's wave decomposition of the raw blob equals the host plan geometry step by
    step — (group, wave) in wave-major order, first dense row, first role row, replicas of the earlier waves."""
    import groups_gen as gg
    from oracle import wave_loop
    case = gg.make_case(seed, n, scarce=seed % 2 == 0)
    states = [wave_loop.GroupState(g) for g in wave_loop.groups_from_blob(case.blob)]
    rc, steps, n_waves, _ = describe(case.blob, n_nodes=case.topo.n, n_domains=len(case.topo.domain_owner))
    assert rc == 0
    assert n_waves == max(len(st.waves) for st in states)
    exp, role_row = [], 0
    group_off = np.cumsum([0] + [sum(st.pending) for st in states])
    for w in range(n_waves):
        for gi, st in enumerate(states):
            if w < len(st.waves):
                i0 = sum(c for wave in st.waves[:w] for _, _, c in wave)
                exp.append((gi, w, int(group_off[gi]) + i0, role_row, i0))
                role_row += len(st.waves[w])
    got = [(int(s[0]), int(s[1]), int(s[4]), int(s[5]), int(s[7])) for s in steps]
    assert got == exp
    assert any(len(wave) == 8 for st in states for wave in st.waves)
