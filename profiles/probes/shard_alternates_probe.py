"""Ranked alternates on node-axis shards (DESIGN.md §3.17) against the world = 1 ranked call, on cfg3-sized fleets
(1 024 mooncake groups, 10 000 nodes) with world = 2 and 4 contexts on one device.  One JSON line per (form, world):
  local_ms    median over ranks and calls of the local half (placement + slab ranking + exchange upload; it ends in a
              device synchronise)
  gather_ms   median of the single-device all-gather (a device concatenation of the ranks' buffers, synchronised)
  merge_ms    median over ranks and calls of the merge half (it ends in a device synchronise)
  world1_ms   median of the world = 1 ranked call on the same fleet, alternated with the sharded calls
  keys_bytes  the exchange buffer of one rank
Every sharded output is checked bit for bit against the world = 1 call.  The lines go to stdout, headed by the card's
name and power limit.  Contexts of one device share it, so local_ms is not the time of a rank on its own GPU.
Usage: python profiles/probes/shard_alternates_probe.py [--calls 10] [--n-alt 8]"""
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


class DevPtr:
    def __init__(self, p, nb):
        self.__cuda_array_interface__ = {"shape": (nb,), "typestr": "|u1", "data": (p, False), "version": 3,
                                         "strides": None}


def placer(topo, **kw):
    e = TopoPlacer(device=0, **kw)
    e.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    return e


def bits(x):
    x = np.asarray(x)
    return x.view(np.uint32) if x.dtype == np.float32 else x


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--n-alt", type=int, default=8)
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    print(json.dumps({"gpu": q[0] if q else "unknown"}))
    n, F = 10000, a.n_alt
    topo = synth.make_topology(n, seed=0)
    e1 = placer(topo)
    gb, _ = B200TopoPodGroupManager(e1).groups_blob(bench.to_plugin(bench.fleet_spec("mooncake", 1024, n, 0)))
    for committed in (False, True):
        one = (lambda: e1.place_groups_committed_ranked(gb, F)) if committed else (lambda: e1.place_groups_ranked(gb, F))
        ref = one()
        for world in (2, 4):
            engs = [placer(topo, rank=r, world=world) for r in range(world)]
            t_loc, t_gat, t_mer, t_one = [], [], [], []
            nbytes = 0
            for it in range(a.calls + 1):   # call 0 warms every shape up
                locs = []
                for e in engs:
                    t0 = time.perf_counter()
                    locs.append(e.shard_place_groups_committed_ranked(gb, F) if committed
                                else e.shard_place_groups_ranked(gb, F))
                    t_loc.append((time.perf_counter() - t0) * 1e3)
                t0 = time.perf_counter()
                allk = torch.cat([torch.as_tensor(DevPtr(l[-2], l[-1]), device="cuda") for l in locs])
                torch.cuda.synchronize()
                t_gat.append((time.perf_counter() - t0) * 1e3)
                for e, l in zip(engs, locs):
                    t0 = time.perf_counter()
                    out = (*l[:-3], *e.shard_alternates_merge(l[-3], allk.data_ptr(), len(l[0]), F))
                    t_mer.append((time.perf_counter() - t0) * 1e3)
                    assert all(np.array_equal(bits(x), bits(y)) for x, y in zip(out, ref)), (committed, world)
                nbytes = locs[0][-1]
                t0 = time.perf_counter()
                one()
                t_one.append((time.perf_counter() - t0) * 1e3)
                if it == 0:
                    t_loc, t_gat, t_mer, t_one = [], [], [], []
            for e in engs:
                e.close()
            print(json.dumps({"form": "committed_ranked" if committed else "ranked", "world": world, "n_alt": F,
                              "groups": int(gb[2]), "replicas": int(gb[4]), "nodes": n,
                              "local_ms": round(float(np.median(t_loc)), 3),
                              "gather_ms": round(float(np.median(t_gat)), 3),
                              "merge_ms": round(float(np.median(t_mer)), 3),
                              "world1_ms": round(float(np.median(t_one)), 3), "keys_bytes": int(nbytes)}))
    e1.close()


if __name__ == "__main__":
    main()
