"""Ranked alternates for leader-worker pods (rbgtopo_place_groups_lw_ranked, DESIGN.md §3.12) on the bench topology
(cfg3: 1 024 mooncake groups, 10 000 nodes) with the prefill role as S = 1, 2 and 4 pods per replica at co-location
level 0 (S = 1: no co-location), F = 0, 2 and 8 alternates, against place_groups_lw on the same input.  One JSON line
per input:
  ms_per_call / lw_ms_per_call   median of >= 20 calls of each (host buffers; every call ends in a device
                                 synchronise), the two entry points alternating
  k_alternates_us                k_alternates' CUDA time in one ranked call (torch.profiler, CUDA activities)
  jobs                           k_alternates CTAs: one per (wave, role) row with a placed pod, one per co-location
                                 domain D_r of the row's replicas when C >= 0
  bytes / k_alternates_gbs       what those jobs read (the row, and the domain vector of each domain condition,
                                 4 bytes per node each) and that over the kernel time
The lines go to stdout, headed by the card's name, power limit and maximum SM clock.
Usage: python profiles/probes/lw_alternates_probe.py [--calls 20]"""
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

MAX_PODS, MAX_ROLES = 32, 8


def jobs_and_bytes(gblob, rp, assign, status, dom0):
    """k_alternates' jobs of one call and the bytes they read, from the pod waves of §3.11 and the placements
    (co-location at level 0 only: dom0 = the level-0 domain of every node)."""
    n = len(dom0)
    gb = np.asarray(gblob, dtype=np.int64)
    jobs = nbytes = 0
    r0 = pod0 = 0
    for g in range(int(gb[2])):
        rec = gb[8 + 12 * g:8 + 12 * (g + 1)]
        q = int(rec[3])
        roles = gb[rec[4]:rec[4] + 4 * q].reshape(q, 4)
        S = [int(rp[r0 + i][0]) for i in range(q)]
        C = [int(rp[r0 + i][1]) for i in range(q)]
        first = np.concatenate([[0], np.cumsum([roles[i, 1] * S[i] for i in range(q)])]).astype(int) + pod0
        waves, cur, npod = [], [], 0   # (role, first replica, replicas), as next_wave splits them
        for ri in range(q):
            if cur and roles[ri, 0] != roles[cur[-1][0], 0]:
                waves.append(cur)
                cur, npod = [], 0
            left, f = int(roles[ri, 1]), 0
            while left > 0:
                take = min(left, (MAX_PODS - npod) // S[ri])
                if take == 0 or len(cur) == MAX_ROLES:
                    waves.append(cur)
                    cur, npod = [], 0
                    continue
                cur.append((ri, f, take))
                npod += take * S[ri]
                left -= take
                f += take
        if cur:
            waves.append(cur)
        if status[g] != 2:
            excl = bool(rec[1] & 1)
            for w in waves:
                for ri, f, reps in w:
                    pods = assign[first[ri] + f * S[ri]:first[ri] + (f + reps) * S[ri]]
                    if not (pods >= 0).any():
                        continue
                    lead = pods[::S[ri]]
                    k = len(set(dom0[lead[lead >= 0]].tolist())) if C[ri] >= 0 else 1
                    jobs += k
                    nbytes += k * n * 4 * (1 + (excl and bool(roles[ri, 3] & 1)) + (C[ri] >= 0))
        r0 += q
        pod0 = int(first[-1])
    return jobs, nbytes


def kernel_us(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return round(sum(e.device_time_total for e in prof.key_averages() if "k_alternates" in e.key), 2)


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
        rp = [(S, 0) if nm == "prefill" and S > 1 else (1, -1) for nm in names]
        for F in (0, 2, 8):
            ranked = lambda: eng.place_groups_lw_ranked(gblob, rp, F)
            plain = lambda: eng.place_groups_lw(gblob, rp)
            a, s, _, _, alt, _ = ranked()
            for _ in range(3):
                plain()
                ranked()
            tr, tl = [], []
            for _ in range(args.calls):
                t0 = time.perf_counter()
                plain()
                t1 = time.perf_counter()
                ranked()
                t2 = time.perf_counter()
                tl.append((t1 - t0) * 1e3)
                tr.append((t2 - t1) * 1e3)
            us = kernel_us(ranked)
            jobs, nbytes = jobs_and_bytes(gblob, rp, a, s, np.asarray(topo.domain))
            print(json.dumps(dict(input="cfg3", prefill_pods=S, colocate=0 if S > 1 else -1, n_alt=F, pods=int(len(a)),
                                  placed=int((a >= 0).sum()), with_alternates=int((alt >= 0).any(axis=1).sum()) if F else 0,
                                  ms_per_call=round(float(np.median(tr)), 3), lw_ms_per_call=round(float(np.median(tl)), 3),
                                  k_alternates_us=us, jobs=jobs, bytes=nbytes,
                                  k_alternates_gbs=round(nbytes / (us * 1e-6) / 1e9, 1) if us > 0 else None)), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
