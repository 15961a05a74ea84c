"""Ranked placement (rbgtopo_place_groups_ranked, DESIGN.md §3.10) on the bench fleets.  One JSON line per input and F:
  ms_per_call / snapshot_ms  median of >= 20 ranked / place_groups calls (host buffers; each call ends in a device
                             synchronise), alternating the two
  k_alternates_us            k_alternates' CUDA time in one ranked call (torch.profiler, CUDA activities)
  k_alternates_gbs           role rows x N x 4 bytes (the rows it reads) over that time
and, on cfg3, a binding simulation: pods bound in blob order, each takes the first of its primary and its F alternates
with room left; `on_hinted_node` counts the pods that land on a hinted node (F = 0: the primary alone).
The lines go to stdout, headed by the card's name, power limit and maximum SM clock.
Usage: python profiles/probes/alternates_probe.py [--calls 20]"""
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

FS = (0, 2, 4, 8)


def role_rows(gblob, assign):
    """(wave, role) rows with a placed replica: what k_alternates reads."""
    b = np.asarray(gblob, dtype=np.int64)
    n = 0
    for g in range(int(b[2])):
        rec = b[8 + 12 * g:8 + 12 * g + 12]
        q, role_off, a0 = int(rec[3]), int(rec[4]), int(rec[8])
        roles = b[role_off:role_off + 4 * q].reshape(q, 4)
        off = np.concatenate([[0], np.cumsum(roles[:, 1])])
        cr, taken = 0, 0
        while cr < q:   # the wave rule of DESIGN.md §3.2
            if roles[cr, 1] - taken <= 0:
                cr, taken = cr + 1, 0
                continue
            level, cnt, entries = roles[cr, 0], 0, 0
            while cr < q and roles[cr, 0] == level and cnt < 32 and entries < 8:
                left = roles[cr, 1] - taken
                if left <= 0:
                    cr, taken = cr + 1, 0
                    continue
                take = min(left, 32 - cnt)
                lo = a0 + off[cr] + taken
                n += int((assign[lo:lo + take] >= 0).any())
                entries += 1
                cnt += take
                taken += take
                if taken == roles[cr, 1]:
                    cr, taken = cr + 1, 0
    return n


def demands(gblob):
    b = np.asarray(gblob, dtype=np.int64)
    out = []
    for g in range(int(b[2])):
        q, role_off = int(b[8 + 12 * g + 3]), int(b[8 + 12 * g + 4])
        for r in range(q):
            out += [int(b[role_off + 4 * r + 2])] * int(b[role_off + 4 * r + 1])
    return np.asarray(out, dtype=np.int64)


def bind(assign, alt, dem, free, F):
    left = free.astype(np.int64).copy()
    landed = 0
    for r in range(len(assign)):
        if assign[r] < 0:
            continue
        for n in [int(assign[r])] + [int(x) for x in alt[r, :F] if x >= 0]:
            if left[n] >= dem[r]:
                left[n] -= dem[r]
                landed += 1
                break
    return landed


def kernel_us(eng, gblob, F):
    import torch
    from torch.profiler import ProfilerActivity, profile
    eng.place_groups_ranked(gblob, F)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.place_groups_ranked(gblob, F)
        torch.cuda.synchronize()
    return sum(e.device_time_total for e in prof.key_averages() if "k_alternates" in e.key)


def run(name, shape, n_groups, n_nodes, calls):
    topo = synth.make_topology(n_nodes, seed=0)
    eng = TopoPlacer(device=0)
    eng.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    gblob, _ = B200TopoPodGroupManager(eng).groups_blob(bench.to_plugin(bench.fleet_spec(shape, n_groups, n_nodes, 0)))
    a0, s0, d0 = eng.place_groups(gblob)
    dem = demands(gblob)
    rows = role_rows(gblob, a0)
    res8 = eng.place_groups_ranked(gblob, 8)
    assert all(np.array_equal(x, y) for x, y in zip(res8[:3], (a0, s0, d0)))
    for F in FS:
        for _ in range(3):
            eng.place_groups(gblob)
            eng.place_groups_ranked(gblob, F)
        ts, tr = [], []
        for _ in range(calls):   # alternating
            t0 = time.perf_counter()
            eng.place_groups(gblob)
            t1 = time.perf_counter()
            eng.place_groups_ranked(gblob, F)
            t2 = time.perf_counter()
            ts.append((t1 - t0) * 1e3)
            tr.append((t2 - t1) * 1e3)
        us = kernel_us(eng, gblob, F)
        line = dict(input=name, groups=n_groups, nodes=n_nodes, replicas=int(len(a0)), F=F, role_rows=rows,
                    ms_per_call=round(float(np.median(tr)), 4), snapshot_ms=round(float(np.median(ts)), 4),
                    k_alternates_us=round(us, 2),
                    k_alternates_gbs=round(rows * n_nodes * 4 / (us * 1e-6) / 1e9, 1) if us > 0 else None)
        if name == "cfg3":
            line["on_hinted_node"] = bind(a0, res8[4], dem, topo.free, F)
            line["placed"] = int((a0 >= 0).sum())
        print(json.dumps(line), flush=True)
    eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    args = ap.parse_args()
    import torch
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(device=torch.cuda.get_device_name(0), nvidia_smi=smi)), flush=True)
    for c in [("cfg3", "mooncake", 1024, 10000), ("cfg4", "fleet8", 1000, 50000)]:
        run(*c, calls=args.calls)


if __name__ == "__main__":
    main()
