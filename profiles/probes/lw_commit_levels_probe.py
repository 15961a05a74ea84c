"""Committed leader-worker batches at exclusive levels (rbgtopo_place_groups_lw_committed on a ctx with
RBGTOPO_CFG_LW_COMMIT_LEVELS, DESIGN.md §3.16) on the bench topology (10 000 nodes) with two partitions installed:
level 1 = racks of 16 nodes, level 2 = hostnames, level 3 = racks of 256 nodes.  10 and 64 mooncake groups, the prefill
role as S = 2 or S = 4 pods per replica, every group but the last exclusive at one key:
  key=0         level 0: the record path of §3.13 (k_score_emit_claims)
  key=0/lists   the same batch with its last (non-exclusive) group's word +10 set to 1: the claim lists of §3.16
                walking level 0 only (k_score_emit_claims_lv), so both kernels can be compared on one batch
  key=rack16, key=hostname, key=rack256   the exclusive groups at levels 1, 2 and 3
One JSON line per input:
  rounds        wave-loop rounds
  ms_per_call   median of `--calls` calls (host buffers; each call ends in a device synchronise)
  emit_us_per_round, assign_us_per_round   CUDA time per round of k_score_emit_claims[_lv] and k_lw_assign
                (torch.profiler, CUDA activities, one call)
  h2d_words     rbgtopo_last_timing h2d_words of the call
The lines go to stdout, headed by the card's name, power limit and maximum SM clock.
Usage: python profiles/probes/lw_commit_levels_probe.py [--calls 20]"""
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
from rbg_b200.blob import STEP_EXCLUSIVE  # noqa: E402
from rbg_b200.engine import TopoPlacer  # noqa: E402
from rbg_b200.plugin import B200TopoPodGroupManager  # noqa: E402


def kernel_us(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    tot = lambda pred: sum(e.device_time_total for e in prof.key_averages() if pred(e.key))
    return tot(lambda k: "k_score_emit_claims" in k), tot(lambda k: "k_lw_assign" in k)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    args = ap.parse_args()
    import torch
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(device=torch.cuda.get_device_name(0), nvidia_smi=smi)), flush=True)
    n = 10000
    topo = synth.make_topology(n, seed=0)
    topo.domain_owner[:] = -1
    eng = TopoPlacer(device=0, lw_committed_levels=True)
    eng.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    lv = np.stack([np.arange(n) // 16, np.arange(n), np.arange(n) // 256]).astype(np.int32)
    eng.set_exclusive_levels(lv, np.zeros((0, 3), np.int32))
    for n_groups in (10, 64):
        base, runs = B200TopoPodGroupManager(eng).groups_blob(bench.to_plugin(bench.fleet_spec("mooncake", n_groups, n, 0)))
        names = [g.rbg.roles[ri].name for g in runs for ri in g.order]
        for S in (2, 4):
            rp = [(S, -1) if nm == "prefill" else (1, -1) for nm in names]
            ref = None
            for key, L in (("0", 0), ("0/lists", 0), ("rack16", 1), ("hostname", 2), ("rack256", 3)):
                gb = np.array(base, dtype=np.int32, copy=True)
                for g in range(n_groups):
                    rec = 8 + 12 * g
                    last = g == n_groups - 1
                    gb[rec + 1] = (gb[rec + 1] | STEP_EXCLUSIVE) if not last else (gb[rec + 1] & ~STEP_EXCLUSIVE)
                    gb[rec + 2] = -1
                    gb[rec + 10] = 1 if (last and key == "0/lists") else (0 if last else L)
                call = lambda: eng.place_groups_lw_committed(gb, rp)
                r = call()
                h2d = eng.last_timing()["h2d_words"]
                if key == "0":
                    ref = r
                elif key == "0/lists":
                    assert all(np.array_equal(x, y) for x, y in zip(r[:3], ref[:3])) and r[3] == ref[3]
                for _ in range(3):
                    call()
                ts = []
                for _ in range(args.calls):
                    t0 = time.perf_counter()
                    call()
                    ts.append((time.perf_counter() - t0) * 1e3)
                emit, assign = kernel_us(call)
                print(json.dumps(dict(input=f"mooncake{n_groups}/{n}", prefill_pods=S, key=key, pods=int(len(r[0])),
                                      placed=int((r[0] >= 0).sum()), rounds=int(r[3]),
                                      ms_per_call=round(float(np.median(ts)), 3),
                                      emit_us_per_round=round(emit / r[3], 2), assign_us_per_round=round(assign / r[3], 2),
                                      h2d_words=int(h2d))), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
