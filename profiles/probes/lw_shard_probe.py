"""Leader-worker placement on node-axis shards (DESIGN.md §3.18) against world = 1, on the bench topology (cfg3: 1 024
mooncake groups, 10 000 nodes) with the prefill role as S = 4 pods per replica at co-location level 0.  World = 2 and
4 contexts (RBGTOPO_CFG_LW_SHARDS) share ONE device, so their numbers are those of ranks sharing one GPU, not per-GPU
times.  One JSON line per (call, world):
  ms_per_call     median over calls of one rank's call (host buffers; each call ends in a device synchronise); world 1
                  and the sharded ranks alternate
  k_lw_assign_us  the CUDA time of k_lw_assign (world 1) or k_lw_assign_repl (world > 1) summed over one call's waves
                  (torch.profiler, CUDA activities, in a run of its own), with k_score_emit's beside it
Every sharded output is checked bit for bit against the world = 1 call.  The lines go to stdout, headed by the card's
name, power limit and maximum SM clock.
--committed adds place_groups_lw_committed, whose rounds on this fleet take seconds to minutes per call.
Usage: python profiles/probes/lw_shard_probe.py [--calls 10] [--committed]"""
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


def placer(topo, **kw):
    e = TopoPlacer(device=0, **kw)
    e.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    return e


def bits(x):
    x = np.asarray(x)
    return x.view(np.uint32) if x.dtype == np.float32 else x


def kernel_us(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    tot = lambda name: round(sum(e.device_time_total for e in prof.key_averages() if name in e.key), 2)
    return tot("k_lw_assign"), tot("k_score_emit")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--committed", action="store_true", help="also the committed form (many rounds per call)")
    args = ap.parse_args()
    import torch
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(device=torch.cuda.get_device_name(0), nvidia_smi=smi)), flush=True)
    n_nodes, n_groups = 10000, 1024
    topo = synth.make_topology(n_nodes, seed=0)
    e1 = placer(topo)
    gblob, runs = B200TopoPodGroupManager(e1).groups_blob(bench.to_plugin(bench.fleet_spec("mooncake", n_groups,
                                                                                         n_nodes, 0)))
    names = [g.rbg.roles[ri].name for g in runs for ri in g.order]
    rp = [(4, 0) if nm == "prefill" else (1, -1) for nm in names]
    for committed in (False, True) if args.committed else (False,):
        call = (lambda e: e.place_groups_lw_committed(gblob, rp)) if committed else (lambda e: e.place_groups_lw(gblob, rp))
        ref = call(e1)
        for world in (2, 4):
            engs = [placer(topo, rank=r, world=world, lw_shards=True) for r in range(world)]
            t1, tw = [], []
            for it in range(args.calls + 1):   # call 0 warms every shape up
                t0 = time.perf_counter()
                call(e1)
                t1.append((time.perf_counter() - t0) * 1e3)
                for e in engs:
                    t0 = time.perf_counter()
                    out = call(e)
                    tw.append((time.perf_counter() - t0) * 1e3)
                    assert all(np.array_equal(bits(x), bits(y)) for x, y in zip(out, ref)), (committed, world)
                if it == 0:
                    t1, tw = [], []
            us1, emit1 = kernel_us(lambda: call(e1))
            usw, emitw = kernel_us(lambda: call(engs[0]))
            form = "lw_committed" if committed else "lw"
            print(json.dumps(dict(call=form, world=1, pods=int(len(ref[0])), placed=int((ref[0] >= 0).sum()),
                                  ms_per_call=round(float(np.median(t1)), 3), k_lw_assign_us=us1,
                                  k_score_emit_us=emit1)), flush=True)
            print(json.dumps(dict(call=form, world=world, ranks_share_one_gpu=True,
                                  ms_per_call=round(float(np.median(tw)), 3), k_lw_assign_us=usw,
                                  k_score_emit_us=emitw)), flush=True)
            for e in engs:
                e.close()
    e1.close()


if __name__ == "__main__":
    main()
