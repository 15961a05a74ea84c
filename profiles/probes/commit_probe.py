"""Committed batches (rbgtopo_place_groups_committed, DESIGN.md §3.8) on the bench fleets and on small batches, with
plentiful and scarce capacity.  Per input, one JSON line:
  ms_per_call        median of >= 20 committed calls (host buffers in and out)
  rounds             selection rounds of the committed call
  plan_us_per_round  median time of one k_plan_group_commit launch (CUDA events, rbgtopo_set_kernel_timing)
  snapshot_ms        median of the same number of rbgtopo_place_groups calls (snapshot semantics, dense matrix included)
  snapshot_overcommitted_nodes / snapshot_unhonourable_hints
                     what the snapshot path's hints ask of the cluster: nodes asked for more than free[n], and the hints
                     that do not fit when the pods are bound in blob order (kube-scheduler places those elsewhere)
  committed_overcommitted_nodes  the same count for the committed call (0 by construction)
Usage: python profiles/probes/commit_probe.py [--calls 20]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from rbg_b200 import synth  # noqa: E402
from rbg_b200.engine import TopoPlacer  # noqa: E402
from rbg_b200.plugin import B200TopoPodGroupManager  # noqa: E402


def demands_in_blob_order(gblob):
    b = np.asarray(gblob, dtype=np.int64)
    out = []
    for g in range(int(b[2])):
        q, role_off = int(b[8 + 12 * g + 3]), int(b[8 + 12 * g + 4])
        for r in range(q):
            out += [int(b[role_off + 4 * r + 2])] * int(b[role_off + 4 * r + 1])
    return np.asarray(out, dtype=np.int64)


def overcommit(assign, dem, free):
    used = np.zeros(len(free), dtype=np.int64)
    ok = assign >= 0
    np.add.at(used, assign[ok], dem[ok])
    nodes = int((used > free).sum())
    left = free.astype(np.int64).copy()
    bad = 0
    for a, d in zip(assign[ok], dem[ok]):   # bound in blob order
        if left[a] >= d:
            left[a] -= d
        else:
            bad += 1
    return nodes, bad


def timed(fn, calls):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(calls):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def run(name, shape, n_groups, n_nodes, scarce, calls):
    topo = synth.make_topology(n_nodes, seed=0, tiers=4, samples_per_tier=5)
    if scarce:   # 80 % of the nodes full, the rest one slot
        rng = np.random.default_rng(1)
        topo.free = np.where(rng.random(n_nodes) < 0.8, 0, np.minimum(topo.free, 1)).astype(np.int32)
    eng = TopoPlacer(device=0)
    eng.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    gblob, _ = B200TopoPodGroupManager(eng).groups_blob(bench.to_plugin(bench.fleet_spec(shape, n_groups, n_nodes, 0)))
    dem = demands_in_blob_order(gblob)
    a_snap, _, _ = eng.place_groups(gblob)
    a_com, s_com, _, rounds = eng.place_groups_committed(gblob)
    snap_nodes, snap_bad = overcommit(a_snap, dem, topo.free)
    com_nodes, com_bad = overcommit(a_com, dem, topo.free)
    ms = timed(lambda: eng.place_groups_committed(gblob), calls)
    snap_ms = timed(lambda: eng.place_groups(gblob), calls)
    eng.set_kernel_timing(True)
    per_round = []
    for _ in range(3):
        eng.place_groups_committed(gblob)
        per_round += list(eng.last_pass_times()[1])
    eng.set_kernel_timing(False)
    eng.close()
    return dict(input=name, groups=n_groups, nodes=n_nodes, scarce=scarce, replicas=int(len(dem)), rounds=int(rounds),
                ms_per_call=round(ms, 4), plan_us_per_round=round(float(np.median(per_round)) * 1e3, 2) if per_round else None,
                snapshot_ms=round(snap_ms, 4), placed_committed=int((a_com >= 0).sum()), placed_snapshot=int((a_snap >= 0).sum()),
                snapshot_overcommitted_nodes=snap_nodes, snapshot_unhonourable_hints=snap_bad,
                committed_overcommitted_nodes=com_nodes, committed_unhonourable_hints=com_bad,
                status_counts=[int((s_com == k).sum()) for k in range(3)])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    args = ap.parse_args()
    import torch
    print(json.dumps(dict(device=torch.cuda.get_device_name(0))), flush=True)
    cases = [("cfg3", "mooncake", 1024, 10000, False), ("cfg4", "fleet8", 1000, 50000, False)]
    for shape in ("mooncake", "fleet8"):
        for ng in (10, 64):
            for scarce in (False, True):
                cases.append((f"{shape}-{ng}", shape, ng, 10000, scarce))
    for c in cases:
        print(json.dumps(run(*c, calls=args.calls)), flush=True)


if __name__ == "__main__":
    main()
