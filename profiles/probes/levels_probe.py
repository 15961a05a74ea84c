"""Placement at exclusive levels (DESIGN.md §3.9, §5): the bench fleet of 1 024 groups x 10 000 nodes with every group
exclusive and at one of three levels — (a) level 0 (the snapshot's domains), (b) a hostname-like level (one node per
domain), (c) a zone-like level of 10 domains — each without and with fixed domains (every group's fixed domain a
random domain of its level).  Per fleet: ms per rbgtopo_place_groups call with host buffers (median of 20, host clock
around the synchronous call) and the device time of k_plan_group launches (torch.profiler CUDA activities, median over the launches of 20
calls, a separate run).  One JSON line per fleet; run on one GPU."""
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

N, G, REPS = 10000, 1024, 20
topo = synth.make_topology(N, seed=0, tiers=4, samples_per_tier=5)
rbgs = bench.build_fleet(G, N)
eng = TopoPlacer(device=0, level_placement=True)
eng.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
base_blob, _ = B200TopoPodGroupManager(eng).groups_blob(rbgs)
rng = np.random.default_rng(0)
levels = np.stack([np.arange(N), (np.arange(N) * 10) // N]).astype(np.int32)   # level 1 hostname-like, level 2 zones
n_dom = [len(topo.domain_owner), N, 10]
gids = [int(base_blob[8 + 12 * g]) for g in range(G)]
# pods of 64 groups on the first 500 nodes (half of zone 0): ownership constrains placement there only
occ = np.array([(int(rng.integers(0, 500)), gids[int(rng.integers(0, 64))], 0) for _ in range(128)], np.int32)
eng.set_exclusive_levels(levels, occ, level_n_domains=n_dom[1:])


def fleet(level, fixed):
    b = np.array(base_blob, dtype=np.int32, copy=True)
    for g in range(G):
        r = 8 + 12 * g
        b[r + 1] |= 1                                    # RBGTOPO_STEP_EXCLUSIVE
        b[r + 10] = level
        b[r + 2] = int(rng.integers(0, n_dom[level])) if fixed else -1
    return b


def plan_kernel_ms(gb):
    """Device time of k_plan_group per place_groups call, from torch.profiler's CUDA activity records."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(REPS):
            eng.place_groups(gb)
    ts = [e.device_time for e in prof.events() if "k_plan_group" in e.name]
    return ts and [x / 1e3 for x in ts] or [float("nan")]


for name, level in (("a_level0", 0), ("b_hostname", 1), ("c_zone10", 2)):
    for fixed in (False, True):
        gb = fleet(level, fixed)
        for _ in range(5):
            eng.place_groups(gb)
        t = []
        for _ in range(REPS):
            t0 = time.perf_counter()
            eng.place_groups(gb)
            t.append((time.perf_counter() - t0) * 1e3)
        sel = plan_kernel_ms(gb)
        a, s, d = eng.place_groups(gb)
        print(json.dumps({"fleet": name, "fixed_domains": fixed, "place_groups_ms": round(float(np.median(t)), 4),
                          "k_plan_group_ms": round(float(np.median(sel)), 4), "placed": int((a >= 0).sum()),
                          "replicas": int(len(a))}), flush=True)
eng.close()
