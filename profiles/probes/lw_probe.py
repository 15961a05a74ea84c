"""Leader-worker placement (rbgtopo_place_groups_lw, DESIGN.md §3.11) on the bench topology (cfg3: 1 024 mooncake groups,
10 000 nodes) with the prefill role as S = 2 and S = 4 pods per replica at co-location level 0, against place_groups
on the same fleet with one pod per replica.  One JSON line per input:
  ms_per_call        median of >= 20 calls (host buffers; each call ends in a device synchronise), the two entry
                     points alternating
  k_lw_assign_us     k_lw_assign's CUDA time summed over one call's waves (torch.profiler, CUDA activities), with
                     k_score_emit's beside it
  pods / placed      pods of the call and how many were placed
The lines go to stdout, headed by the card's name, power limit and maximum SM clock.
Usage: python profiles/probes/lw_probe.py [--calls 20]"""
import argparse
import json
import os
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


def kernel_us(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    tot = lambda name: round(sum(e.device_time_total for e in prof.key_averages() if name in e.key), 2)
    return tot("k_lw_assign"), tot("k_score_emit"), tot("k_emit_rows"), tot("k_plan_group")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    args = ap.parse_args()
    import torch
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(device=torch.cuda.get_device_name(0), nvidia_smi=smi)), flush=True)
    n_nodes, n_groups = 10000, 1024
    topo = synth.make_topology(n_nodes, seed=0)
    eng = TopoPlacer(device=0)
    eng.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    gblob, runs = B200TopoPodGroupManager(eng).groups_blob(bench.to_plugin(bench.fleet_spec("mooncake", n_groups,
                                                                                             n_nodes, 0)))
    names = [g.rbg.roles[ri].name for g in runs for ri in g.order]
    for S in (1, 2, 4):
        rp = [(S, 0) if nm == "prefill" else (1, -1) for nm in names]
        if S == 1:
            rp = [(1, -1)] * len(names)
        lw_call = lambda: eng.place_groups_lw(gblob, rp)
        a, _, _ = lw_call()
        for _ in range(3):
            eng.place_groups(gblob)
            lw_call()
        tl, tp = [], []
        for _ in range(args.calls):
            t0 = time.perf_counter()
            eng.place_groups(gblob)
            t1 = time.perf_counter()
            lw_call()
            t2 = time.perf_counter()
            tp.append((t1 - t0) * 1e3)
            tl.append((t2 - t1) * 1e3)
        lw_us, score_us, _, _ = kernel_us(lw_call)
        _, _, emit_us, plan_us = kernel_us(lambda: eng.place_groups(gblob))
        print(json.dumps(dict(input="cfg3", prefill_pods=S, colocate=0 if S > 1 else -1, pods=int(len(a)),
                              placed=int((a >= 0).sum()), ms_per_call=round(float(np.median(tl)), 3),
                              place_groups_ms=round(float(np.median(tp)), 3), k_lw_assign_us=lw_us,
                              k_score_emit_us=score_us, place_groups_k_emit_rows_us=emit_us,
                              place_groups_k_plan_group_us=plan_us)), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
