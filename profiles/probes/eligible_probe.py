"""Node eligibility (rbgtopo_place_groups_eligible, DESIGN.md §3.19) on the bench topology (cfg3: 1 024 mooncake
groups, 10 000 nodes), prefill as S = 2 pods per replica at co-location level 0, every node in one of 4 classes and every
mask admitting all of them, against the calls it reduces to.  One JSON line per pair, the two calls alternating:
  a_ms / b_ms               median of --calls host-buffer calls (each ends in a device synchronise)
  a_kernel_us / b_kernel_us median over --reps profiled calls of the dense-row kernel's CUDA time summed over the
                            call's waves (torch.profiler, CUDA activities): k_score_emit against k_score_emit_elig
The pairs: place_groups_lw vs place_groups_eligible (role_pods given), and place_groups (the device-resident plan) vs
place_groups_eligible with role_pods NULL (the price of routing a plain group through the row-reading loop).
The lines go to stdout, headed by the card's name, power limit and maximum SM clock.
Usage: python profiles/probes/eligible_probe.py [--calls 20] [--reps 5]"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from rbg_b200 import synth  # noqa: E402
from rbg_b200.engine import TopoPlacer  # noqa: E402
from rbg_b200.plugin import B200TopoPodGroupManager  # noqa: E402


def kernel_us(fn, name):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    pat = re.compile(r"(^|\W)" + name + r"[<(]")   # k_score_emit( but not k_score_emit_elig(
    return sum(e.device_time_total for e in prof.key_averages() if pat.search(e.key))


def pair(label, fa, fb, ka, kb, calls, reps):
    for _ in range(3):
        fa()
        fb()
    ta, tb = [], []
    for _ in range(calls):
        t0 = time.perf_counter()
        fa()
        t1 = time.perf_counter()
        fb()
        t2 = time.perf_counter()
        ta.append((t1 - t0) * 1e3)
        tb.append((t2 - t1) * 1e3)
    ua, ub = [], []
    for _ in range(reps):
        ua.append(kernel_us(fa, ka))
        ub.append(kernel_us(fb, kb))
    print(json.dumps(dict(pair=label, a_ms=round(float(np.median(ta)), 3), b_ms=round(float(np.median(tb)), 3),
                          a_kernel=ka, a_kernel_us=round(float(np.median(ua)), 2), b_kernel=kb,
                          b_kernel_us=round(float(np.median(ub)), 2))), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(device=torch.cuda.get_device_name(0), nvidia_smi=smi)), flush=True)
    n_nodes, n_groups = 10000, 1024
    topo = synth.make_topology(n_nodes, seed=0)
    eng = TopoPlacer(device=0)
    eng.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    eng.set_node_classes(np.arange(n_nodes, dtype=np.int32) % 4, 4)
    gblob, runs = B200TopoPodGroupManager(eng).groups_blob(bench.to_plugin(bench.fleet_spec("mooncake", n_groups,
                                                                                             n_nodes, 0)))
    names = [g.rbg.roles[ri].name for g in runs for ri in g.order]
    rp = [(2, 0) if nm == "prefill" else (1, -1) for nm in names]
    full = np.full(len(names), 0xF, np.uint64)
    a = eng.place_groups_eligible(gblob, rp, full)
    b = eng.place_groups_lw(gblob, rp)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    pair("place_groups_lw|place_groups_eligible", lambda: eng.place_groups_lw(gblob, rp),
         lambda: eng.place_groups_eligible(gblob, rp, full), "k_score_emit", "k_score_emit_elig", args.calls, args.reps)
    pair("place_groups|place_groups_eligible(role_pods=NULL)", lambda: eng.place_groups(gblob),
         lambda: eng.place_groups_eligible(gblob, None, full), "k_emit_rows", "k_score_emit_elig", args.calls, args.reps)
    eng.close()


if __name__ == "__main__":
    main()
