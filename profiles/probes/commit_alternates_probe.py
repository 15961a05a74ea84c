"""Ranked alternates of committed batches (rbgtopo_place_groups_committed_ranked, DESIGN.md §3.14) on the bench fleets.
One JSON line per input and F:
  ms_per_call / committed_ms   median of >= 20 ranked-committed / place_groups_committed calls (host buffers; each call
                               ends in a device synchronise), alternating the two
  emit_us / alt_us             CUDA time of the replay's k_score_emit and of k_alternates_commit in one call
                               (torch.profiler, CUDA activities)
  emit_gbs / alt_gbs           rows x N x 4 bytes (the rows k_score_emit writes / k_alternates_commit reads) over it
  snapshot_alt_no_room         of the alternates place_groups_ranked gives the same batch (snapshot semantics), the
                               share that has no room for the replica once the committed batch is placed
  committed_alt_no_room        the same share for the new call's alternates (0 by construction)
The lines go to stdout, headed by the card's name, power limit and maximum SM clock.
Usage: python profiles/probes/commit_alternates_probe.py [--calls 20]"""
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


def replay_rows(gblob, assign, status):
    """(rows k_score_emit writes, rows k_alternates_commit reads): every role row of a (group, wave) with a placed
    replica, and those of its roles with one (§3.14; the wave rule of §3.2)."""
    b = np.asarray(gblob, dtype=np.int64)
    emit = alt = 0
    for g in range(int(b[2])):
        if status[g] == 2:
            continue
        rec = b[8 + 12 * g:8 + 12 * g + 12]
        q, role_off, a0 = int(rec[3]), int(rec[4]), int(rec[8])
        roles = b[role_off:role_off + 4 * q].reshape(q, 4)
        off = np.concatenate([[0], np.cumsum(roles[:, 1])])
        cr, taken = 0, 0
        while cr < q:
            if roles[cr, 1] - taken <= 0:
                cr, taken = cr + 1, 0
                continue
            level, cnt, placed = roles[cr, 0], 0, []
            while cr < q and roles[cr, 0] == level and cnt < 32 and len(placed) < 8:
                left = roles[cr, 1] - taken
                if left <= 0:
                    cr, taken = cr + 1, 0
                    continue
                take = min(left, 32 - cnt)
                lo = a0 + off[cr] + taken
                placed.append(bool((assign[lo:lo + take] >= 0).any()))
                cnt += take
                taken += take
                if taken == roles[cr, 1]:
                    cr, taken = cr + 1, 0
            if any(placed):
                emit += len(placed)
                alt += sum(placed)
    return emit, alt


def demands(gblob):
    b = np.asarray(gblob, dtype=np.int64)
    out = []
    for g in range(int(b[2])):
        q, role_off = int(b[8 + 12 * g + 3]), int(b[8 + 12 * g + 4])
        for r in range(q):
            out += [int(b[role_off + 4 * r + 2])] * int(b[role_off + 4 * r + 1])
    return np.asarray(out, dtype=np.int64)


def no_room(alt, assign, dem, free):
    """Share of the alternates with no room for their replica once the committed batch (assign) is placed."""
    used = np.zeros(len(free), dtype=np.int64)
    ok = assign >= 0
    np.add.at(used, assign[ok], dem[ok])
    room = free.astype(np.int64) - used
    rows, cols = np.nonzero(alt >= 0)
    if len(rows) == 0:
        return None, 0
    bad = room[alt[rows, cols]] < dem[rows]
    return round(float(bad.mean()), 4), int(len(rows))


def kernel_us(eng, gblob, F):
    import torch
    from torch.profiler import ProfilerActivity, profile
    eng.place_groups_committed_ranked(gblob, F)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.place_groups_committed_ranked(gblob, F)
        torch.cuda.synchronize()
    ka = prof.key_averages()
    emit = sum(e.device_time_total for e in ka if "k_score_emit" in e.key)
    alt = sum(e.device_time_total for e in ka if "k_alternates_commit" in e.key)
    return emit, alt


def run(name, shape, n_groups, n_nodes, calls):
    topo = synth.make_topology(n_nodes, seed=0)
    eng = TopoPlacer(device=0)
    eng.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    gblob, _ = B200TopoPodGroupManager(eng).groups_blob(bench.to_plugin(bench.fleet_spec(shape, n_groups, n_nodes, 0)))
    a0, s0, d0, r0 = eng.place_groups_committed(gblob)
    dem = demands(gblob)
    emit_rows, alt_rows = replay_rows(gblob, a0, s0)
    for F in FS:
        res = eng.place_groups_committed_ranked(gblob, F)
        assert all(np.array_equal(x, y) for x, y in zip(res[:3], (a0, s0, d0))) and res[3] == r0
        for _ in range(3):
            eng.place_groups_committed(gblob)
            eng.place_groups_committed_ranked(gblob, F)
        tc, tr = [], []
        for _ in range(calls):   # alternating
            t0 = time.perf_counter()
            eng.place_groups_committed(gblob)
            t1 = time.perf_counter()
            eng.place_groups_committed_ranked(gblob, F)
            t2 = time.perf_counter()
            tc.append((t1 - t0) * 1e3)
            tr.append((t2 - t1) * 1e3)
        emit_us, alt_us = kernel_us(eng, gblob, F)
        line = dict(input=name, groups=n_groups, nodes=n_nodes, replicas=int(len(a0)), placed=int((a0 >= 0).sum()),
                    rounds=r0, F=F, emit_rows=emit_rows, alt_rows=alt_rows,
                    ms_per_call=round(float(np.median(tr)), 3), committed_ms=round(float(np.median(tc)), 3),
                    emit_us=round(emit_us, 1), alt_us=round(alt_us, 1),
                    emit_gbs=round(emit_rows * n_nodes * 4 / (emit_us * 1e-6) / 1e9, 1) if emit_us > 0 else None,
                    alt_gbs=round(alt_rows * n_nodes * 4 / (alt_us * 1e-6) / 1e9, 1) if alt_us > 0 else None)
        if F > 0:
            snap = eng.place_groups_ranked(gblob, F)
            line["snapshot_alt_no_room"], line["snapshot_alts"] = no_room(snap[4], a0, dem, topo.free)
            line["committed_alt_no_room"], line["committed_alts"] = no_room(res[5], a0, dem, topo.free)
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
