"""Node eligibility in committed batches (rbgtopo_place_groups_eligible_committed, DESIGN.md §3.20) against
place_groups_lw_committed on the 10- and 64-group mooncake batches of §5 (10 000-node bench topology, prefill as S = 4
pods per replica co-located at level 0), every node in one of 4 classes and every mask admitting all of them; the
outputs, rounds included, are asserted equal.  One JSON line per batch, the two calls alternating:
  a_ms / b_ms               median of --calls host-buffer calls (each ends in a device synchronise)
  a_kernel_us / b_kernel_us median over --reps profiled calls of the dense-row kernel's CUDA time summed over the call's
                            waves (torch.profiler, CUDA activities): k_score_emit_claims against
                            k_score_emit_claims_elig; *_per_round_us divides it by the call's rounds
The lines go to stdout, headed by the card's name, power limit and maximum SM clock.
Usage: python profiles/probes/eligible_commit_probe.py [--calls 20] [--reps 5]"""
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
    pat = re.compile(r"(^|\W)" + name + r"[<(]")   # k_score_emit_claims( but not k_score_emit_claims_elig(
    return sum(e.device_time_total for e in prof.key_averages() if pat.search(e.key))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(device=torch.cuda.get_device_name(0), nvidia_smi=smi)), flush=True)
    n_nodes = 10000
    topo = synth.make_topology(n_nodes, seed=0)
    eng = TopoPlacer(device=0)
    eng.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    eng.set_node_classes(np.arange(n_nodes, dtype=np.int32) % 4, 4)
    for n_groups in (10, 64):
        gblob, runs = B200TopoPodGroupManager(eng).groups_blob(
            bench.to_plugin(bench.fleet_spec("mooncake", n_groups, n_nodes, 0)))
        names = [g.rbg.roles[ri].name for g in runs for ri in g.order]
        rp = [(4, 0) if nm == "prefill" else (1, -1) for nm in names]
        full = np.full(len(names), 0xF, np.uint64)
        fa = lambda: eng.place_groups_lw_committed(gblob, rp)
        fb = lambda: eng.place_groups_eligible_committed(gblob, rp, full)
        a, b = fa(), fb()
        assert all(np.array_equal(x, y) for x, y in zip(a[:3], b[:3])) and a[3] == b[3]
        for _ in range(3):
            fa()
            fb()
        ta, tb = [], []
        for _ in range(args.calls):
            t0 = time.perf_counter()
            fa()
            t1 = time.perf_counter()
            fb()
            t2 = time.perf_counter()
            ta.append((t1 - t0) * 1e3)
            tb.append((t2 - t1) * 1e3)
        ua, ub = [], []
        for _ in range(args.reps):
            ua.append(kernel_us(fa, "k_score_emit_claims"))
            ub.append(kernel_us(fb, "k_score_emit_claims_elig"))
        ka, kb = float(np.median(ua)), float(np.median(ub))
        print(json.dumps(dict(input=f"mooncake{n_groups}/{n_nodes}", prefill_pods=4, colocate=0, rounds=int(a[3]),
                              pods=int(len(a[0])), placed=int((a[0] >= 0).sum()),
                              a="place_groups_lw_committed", b="place_groups_eligible_committed",
                              a_ms=round(float(np.median(ta)), 3), b_ms=round(float(np.median(tb)), 3),
                              a_ms_range=[round(float(min(ta)), 3), round(float(max(ta)), 3)],
                              b_ms_range=[round(float(min(tb)), 3), round(float(max(tb)), 3)],
                              a_kernel="k_score_emit_claims", a_kernel_us=round(ka, 2),
                              a_per_round_us=round(ka / max(a[3], 1), 2),
                              b_kernel="k_score_emit_claims_elig", b_kernel_us=round(kb, 2),
                              b_per_round_us=round(kb / max(a[3], 1), 2))), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
