"""Committed batches at exclusive levels (rbgtopo_place_groups_committed with RBGTOPO_CFG_COMMIT_LEVELS, DESIGN.md §3.8 /
§3.9).  One JSON line per input:
  --mode level0   the level-0 rows of commit_probe.py (cfg3, cfg4, mooncake-64 scarce) on a ctx without the new flag:
                  run it once per library (RBGTOPO_LIB selects one) and alternate, to compare builds
  --mode levels   bench mooncake fleets of 64 and 1 024 groups, every group exclusive at level g % 4 of a 10 000-node
                  snapshot (level 1 hostname, level 2 ten zones, level 3 racks of ~40 nodes inside the zones), records of
                  one outside gid on 2 % of the nodes keyed at levels 0 and 1 (a zone-keyed record would block its
                  whole zone for every group), with and without fixed domains at the groups' levels
Fields: ms_per_call (median of --calls calls), rounds, plan_us_per_round (median k_plan_group_commit launch, CUDA
events), the card's name and power limit.
Usage: python profiles/probes/commit_levels_probe.py --mode levels [--calls 10]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench  # noqa: E402
from commit_probe import timed  # noqa: E402
from rbg_b200 import synth  # noqa: E402
from rbg_b200.blob import ROLE_EXCLUSIVE, STEP_EXCLUSIVE  # noqa: E402
from rbg_b200.engine import TopoPlacer  # noqa: E402
from rbg_b200.plugin import B200TopoPodGroupManager  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers are still worth printing
        q = f"unknown ({e})"
    return dict(card=q, lib=os.environ.get("RBGTOPO_LIB", "tree"))


def per_round(eng, fn):
    eng.set_kernel_timing(True)
    out = []
    for _ in range(3):
        fn()
        out += list(eng.last_pass_times()[1])
    eng.set_kernel_timing(False)
    return round(float(np.median(out)) * 1e3, 2) if out else None


def level0(name, shape, n_groups, n_nodes, scarce, calls):
    topo = synth.make_topology(n_nodes, seed=0, tiers=4, samples_per_tier=5)
    if scarce:
        rng = np.random.default_rng(1)
        topo.free = np.where(rng.random(n_nodes) < 0.8, 0, np.minimum(topo.free, 1)).astype(np.int32)
    eng = TopoPlacer(device=0)
    eng.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    gb, _ = B200TopoPodGroupManager(eng).groups_blob(bench.to_plugin(bench.fleet_spec(shape, n_groups, n_nodes, 0)))
    a, s, d, rounds = eng.place_groups_committed(gb)
    ms = timed(lambda: eng.place_groups_committed(gb), calls)
    pr = per_round(eng, lambda: eng.place_groups_committed(gb))
    eng.close()
    return dict(mode="level0", input=name, rounds=int(rounds), ms_per_call=round(ms, 4), plan_us_per_round=pr,
                placed=int((a >= 0).sum()), **card())


def levels(n_groups, fixed, calls, n_nodes=10000):
    topo = synth.make_topology(n_nodes, seed=0, tiers=4, samples_per_tier=5)
    topo.domain_owner[:] = -1
    rng = np.random.default_rng(7)
    zone = rng.integers(0, 10, n_nodes)
    rack = zone * 25 + rng.integers(0, 25, n_nodes)
    _, rack = np.unique(rack, return_inverse=True)
    lv = np.stack([np.arange(n_nodes), zone, rack]).astype(np.int32)
    nd = [n_nodes, 10, int(rack.max()) + 1]
    occ = np.stack([rng.choice(n_nodes, n_nodes // 50, replace=False), np.full(n_nodes // 50, 99999),
                    rng.integers(0, 2, n_nodes // 50)], axis=1).astype(np.int32)  # NVLink- and hostname-keyed
    eng = TopoPlacer(device=0, committed_levels=True)
    eng.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    eng.set_exclusive_levels(lv, occ, level_n_domains=nd)
    gb, _ = B200TopoPodGroupManager(eng).groups_blob(bench.to_plugin(bench.fleet_spec("mooncake", n_groups, n_nodes, 0)))
    gb = np.array(gb, dtype=np.int32, copy=True)
    nds = [len(topo.domain_owner)] + nd
    for g in range(n_groups):
        rec = 8 + 12 * g
        L = g % 4
        gb[rec + 1] |= STEP_EXCLUSIVE
        gb[rec + 10] = L
        gb[rec + 2] = int(rng.integers(0, nds[L])) if fixed and g % 3 == 0 else -1
        q, roff = int(gb[rec + 3]), int(gb[rec + 4])
        for r in range(q):
            gb[roff + 4 * r + 3] |= ROLE_EXCLUSIVE
    a, s, d, rounds = eng.place_groups_committed(gb)
    ms = timed(lambda: eng.place_groups_committed(gb), calls)
    pr = per_round(eng, lambda: eng.place_groups_committed(gb))
    eng.close()
    return dict(mode="levels", groups=n_groups, fixed=fixed, rounds=int(rounds), ms_per_call=round(ms, 4),
                plan_us_per_round=pr, placed=int((a >= 0).sum()), replicas=int(len(a)),
                status_counts=[int((s == k).sum()) for k in range(3)], **card())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", choices=["level0", "levels"], required=True)
    ap.add_argument("--calls", type=int, default=20)
    args = ap.parse_args()
    if args.mode == "level0":
        for c in [("cfg3", "mooncake", 1024, 10000, False), ("cfg4", "fleet8", 1000, 50000, False),
                  ("mooncake-64-scarce", "mooncake", 64, 10000, True)]:
            print(json.dumps(level0(*c, calls=args.calls)), flush=True)
    else:
        for ng in (64, 1024):
            for fixed in (False, True):
                print(json.dumps(levels(ng, fixed, args.calls)), flush=True)


if __name__ == "__main__":
    main()
