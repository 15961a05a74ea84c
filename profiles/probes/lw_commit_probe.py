"""Committed leader-worker batches (rbgtopo_place_groups_lw_committed, DESIGN.md §3.13) on the bench topology (10 000
nodes): 10 and 64 mooncake groups with the prefill role as S = 2 and S = 4 pods per replica co-located at level 0, with
the snapshot's capacity and with 80 % of the nodes full.  One JSON line per input:
  rounds              wave-loop rounds of the committed call
  ms_per_call         median of `--calls` calls (host buffers; each call ends in a device synchronise), the committed
                      call and place_groups_lw alternating (lw_ms_per_call)
  per_round_us        k_score_emit_claims + k_lw_assign CUDA time of one call over its rounds (torch.profiler, CUDA
                      activities), and the two kernels apart over the whole call
  lw_over_nodes       place_groups_lw on the same blob: nodes asked for more than free[n] by the batch's hints
  lw_misfit_hints     ... and its placed pods that do not fit, taking the pods in blob order
  (committed_over_nodes / committed_misfit_hints: the same for the committed call; both must be 0)
The lines go to stdout, headed by the card's name, power limit and maximum SM clock.
Usage: python profiles/probes/lw_commit_probe.py [--calls 20]"""
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


def pod_demand(gblob, rp):
    """Demand of every pod in assign order (group, role, ordinal, k)."""
    out, k = [], 0
    for g in range(int(gblob[2])):
        rec = 8 + 12 * g
        q, off = int(gblob[rec + 3]), int(gblob[rec + 4])
        for i in range(q):
            pending, demand = int(gblob[off + 4 * i + 1]), int(gblob[off + 4 * i + 2])
            out += [demand] * (pending * rp[k + i][0])
        k += q
    return np.asarray(out, dtype=np.int64)


def overcommit(free, assign, demand):
    """(nodes asked for more than free[n], placed pods that do not fit when taken in blob order)."""
    used = np.zeros(len(free), dtype=np.int64)
    misfit = 0
    for node, dem in zip(assign, demand):
        if node >= 0:
            used[node] += dem
            misfit += int(used[node] > free[node])
    return int((used > free).sum()), misfit


def kernel_us(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    tot = lambda name: round(sum(e.device_time_total for e in prof.key_averages() if name in e.key), 2)
    return tot("k_score_emit_claims"), tot("k_lw_assign")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    args = ap.parse_args()
    import torch
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(device=torch.cuda.get_device_name(0), nvidia_smi=smi)), flush=True)
    n_nodes = 10000
    for scarce in (False, True):
        topo = synth.make_topology(n_nodes, seed=0)
        if scarce:
            full = np.random.default_rng(1).random(n_nodes) < 0.8
            topo.free = np.where(full, 0, topo.free).astype(np.int32)
        eng = TopoPlacer(device=0)
        eng.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
        for n_groups in (10, 64):
            gblob, runs = B200TopoPodGroupManager(eng).groups_blob(
                bench.to_plugin(bench.fleet_spec("mooncake", n_groups, n_nodes, 0)))
            names = [g.rbg.roles[ri].name for g in runs for ri in g.order]
            for S in (2, 4):
                rp = [(S, 0) if nm == "prefill" else (1, -1) for nm in names]
                dem = pod_demand(gblob, rp)
                commit = lambda: eng.place_groups_lw_committed(gblob, rp)
                snap = lambda: eng.place_groups_lw(gblob, rp)
                a, _, _, rounds = commit()
                b, _, _ = snap()
                for _ in range(3):
                    commit()
                    snap()
                tc, ts = [], []
                for _ in range(args.calls):
                    t0 = time.perf_counter()
                    commit()
                    t1 = time.perf_counter()
                    snap()
                    t2 = time.perf_counter()
                    tc.append((t1 - t0) * 1e3)
                    ts.append((t2 - t1) * 1e3)
                emit_us, assign_us = kernel_us(commit)
                co, cm = overcommit(topo.free, a, dem)
                lo_, lm = overcommit(topo.free, b, dem)
                print(json.dumps(dict(input=f"mooncake{n_groups}/{n_nodes}", scarce=scarce, prefill_pods=S, colocate=0,
                                      pods=int(len(a)), placed=int((a >= 0).sum()), rounds=rounds,
                                      ms_per_call=round(float(np.median(tc)), 3),
                                      lw_ms_per_call=round(float(np.median(ts)), 3),
                                      per_round_us=round((emit_us + assign_us) / max(rounds, 1), 2),
                                      k_score_emit_claims_us=emit_us, k_lw_assign_us=assign_us,
                                      committed_over_nodes=co, committed_misfit_hints=cm,
                                      lw_over_nodes=lo_, lw_misfit_hints=lm, lw_placed=int((b >= 0).sum()))),
                      flush=True)
        eng.close()


if __name__ == "__main__":
    main()
