"""CPU: the oracle-side level/wave loop (oracle/wave_loop.py, what bench.py's checker and reference
arm use) against the plugin mirror's loop (rbg_b200/plugin.py) — two independent restatements of
the role order, the wave rule, the pair matrix, `need` and the BLOB wire format must produce the
same step batches word for word and the same results."""
import numpy as np
import pytest

import bench
from oracle import wave_loop
from rbg_b200 import synth
from rbg_b200.plugin import B200TopoPodGroupManager
from test_plugin_host import OraclePlacer


@pytest.mark.parametrize("shape,n_groups,n", [("mooncake", 12, 1500), ("fleet8", 9, 700), ("pd144", 5, 600)])
def test_wave_blobs_and_results_match_the_plugin_mirror(shape, n_groups, n):
    topo = synth.make_topology(n, seed=4, tiers=3)
    specs = bench.fleet_spec(shape, n_groups, n, seed=2)
    pl = OraclePlacer(topo)
    ref = B200TopoPodGroupManager(pl).reconcile_pod_groups_by_waves(bench.to_plugin(specs))
    states, blobs = wave_loop.run_fleet(topo, bench.to_oracle(specs))
    assert len(blobs) == len(pl.blobs)
    for a, b in zip(blobs, pl.blobs):
        assert np.array_equal(a, b)
    for st, r in zip(states, ref):
        res = st.result()
        assert res["nodes"] == r.nodes and res["status"] == r.status and res["domain"] == r.domain
    # the plugin's own GROUPS blob, decoded by the oracle alone (explicit levels, pair matrix, anchor counts)
    gblob, _ = B200TopoPodGroupManager(pl).groups_blob(bench.to_plugin(specs))
    decoded, _ = wave_loop.run_fleet(topo, wave_loop.groups_from_blob(gblob))
    for st, d in zip(states, decoded):
        assert d.assign_in_group_order() == st.assign_in_group_order()
        assert (d.result()["status"], d.result()["domain"]) == (st.result()["status"], st.result()["domain"])
        assert [[c for _, _, c in w] for w in d.waves] == [[c for _, _, c in w] for w in st.waves]


def test_big_gang_exclusive_groups():
    from oracle.wave_loop import OGroup, ORole
    from rbg_b200.plugin import EXCLUSIVE_TOPOLOGY_KEY, GANG_SCHEDULING_KEY, RoleBasedGroup, RoleSpec
    topo = synth.make_topology(2048, seed=9, tiers=4, owned_frac=0.2)
    og, pg = [], []
    for g in range(6):
        roles = [("decode", 3, (), 1), ("prefill", 41 if g % 2 else 4, (), 1), ("router", 1, ("decode", "prefill"), 0)]
        og.append(OGroup(f"g{g}", g, [ORole(*r) for r in roles], rules=[("prefill", "decode")], exclusive=g % 3 == 0,
                         gang=g % 2 == 0, placed=[("decode", 8 * g)] if g % 2 else [], current={"decode": 1} if g % 2 else {}))
        ann = {}
        if g % 3 == 0:
            ann[EXCLUSIVE_TOPOLOGY_KEY] = "zone"
        if g % 2 == 0:
            ann[GANG_SCHEDULING_KEY] = "true"
        pg.append(RoleBasedGroup("ns", f"g{g}", [RoleSpec(*r) for r in roles], annotations=ann, gid=g,
                                 policy_rules=[("prefill", "decode")], placed=[("decode", 8 * g)] if g % 2 else [],
                                 current={"decode": 1} if g % 2 else {}))
    pl = OraclePlacer(topo)
    ref = B200TopoPodGroupManager(pl).reconcile_pod_groups_by_waves(pg)
    states, blobs = wave_loop.run_fleet(topo, og)
    assert len(blobs) == len(pl.blobs) and all(np.array_equal(a, b) for a, b in zip(blobs, pl.blobs))
    for st, r in zip(states, ref):
        res = st.result()
        assert res["nodes"] == r.nodes and res["status"] == r.status and res["domain"] == r.domain


def test_reference_arm_does_not_load_the_product_library():
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0",
                        "--ref-groups", "4", "--groups", "8", "--nodes", "500"], cwd=root, capture_output=True, text=True,
                       timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    d = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("{")][0])
    assert d["product_so_loaded"] is False
