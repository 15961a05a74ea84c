"""Ranked alternates of committed leader-worker batches (rbgtopo_place_groups_lw_committed_ranked, DESIGN.md §3.15) on
the bench topology (10 000 nodes): 10 and 64 mooncake groups with the prefill role as S = 4 pods per replica
co-located at level 0, n_alt = 8.  One JSON line per input:
  rounds              wave-loop rounds (the same for both calls)
  ms_per_call         median of `--calls` calls of the ranked call (host buffers; each call ends in a device
                      synchronise), alternating with place_groups_lw_committed on the same blob (commit_ms_per_call)
  launches            rbgtopo_last_timing launches of the ranked call, and of place_groups_lw_committed
  replay_chunks       (launches - commit_launches) / 2: one replay score launch and one ranking launch per chunk
  rank_us             CUDA time of the ranking in one call (torch.profiler, CUDA activities): the replay's k_score_emit
                      and k_alternates_commit*, each also apart
  alternates          alternates listed over all pods
The lines go to stdout, headed by the card's name, power limit and maximum SM clock.
Usage: python profiles/probes/lw_commit_alternates_probe.py [--calls 20]"""
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
    tot = lambda pred: round(sum(e.device_time_total for e in prof.key_averages() if pred(e.key)), 2)
    # k_score_emit without the _claims variant of the rounds: the replay
    emit = tot(lambda k: "k_score_emit" in k and "k_score_emit_claims" not in k)
    alt = tot(lambda k: "k_alternates_commit" in k)
    return emit, alt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    args = ap.parse_args()
    import torch
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(device=torch.cuda.get_device_name(0), nvidia_smi=smi)), flush=True)
    n_nodes, F = 10000, 8
    topo = synth.make_topology(n_nodes, seed=0)
    eng = TopoPlacer(device=0)
    eng.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    for n_groups in (10, 64):
        gblob, runs = B200TopoPodGroupManager(eng).groups_blob(
            bench.to_plugin(bench.fleet_spec("mooncake", n_groups, n_nodes, 0)))
        names = [g.rbg.roles[ri].name for g in runs for ri in g.order]
        rp = [(4, 0) if nm == "prefill" else (1, -1) for nm in names]
        ranked = lambda: eng.place_groups_lw_committed_ranked(gblob, rp, F)
        commit = lambda: eng.place_groups_lw_committed(gblob, rp)
        b = commit()
        commit_launches = eng.last_timing()["launches"]
        r = ranked()
        launches = eng.last_timing()["launches"]
        assert all(np.array_equal(x, y) for x, y in zip(r[:3], b[:3])) and r[3] == b[3]
        for _ in range(3):
            ranked()
            commit()
        tr, tc = [], []
        for _ in range(args.calls):
            t0 = time.perf_counter()
            ranked()
            t1 = time.perf_counter()
            commit()
            t2 = time.perf_counter()
            tr.append((t1 - t0) * 1e3)
            tc.append((t2 - t1) * 1e3)
        emit_us, alt_us = kernel_us(ranked)
        print(json.dumps(dict(input=f"mooncake{n_groups}/{n_nodes}", prefill_pods=4, colocate=0, n_alt=F,
                              pods=int(len(r[0])), placed=int((r[0] >= 0).sum()), rounds=r[3],
                              ms_per_call=round(float(np.median(tr)), 3),
                              commit_ms_per_call=round(float(np.median(tc)), 3),
                              launches=launches, commit_launches=commit_launches,
                              replay_chunks=(launches - commit_launches) // 2,
                              rank_us=round(emit_us + alt_us, 2), replay_emit_us=emit_us, k_alternates_us=alt_us,
                              alternates=int((r[5] >= 0).sum()))), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
