"""GPU: the plugin with alternates on a world = 2 pair of placers (two contexts on one device, each behind its own
B200TopoPodGroupManager, reconciling from two threads).  The managers' all-gather is a rendezvous that concatenates
the two exchange buffers on the device.  Hints and alternates must equal those of the world = 1 plugin, for snapshot
and committed batches."""
import threading

import pytest

from rbg_b200 import synth
from rbg_b200.engine import TopoPlacer
from rbg_b200.plugin import B200TopoPodGroupManager
from test_gpu_shard_alternates import gather

pytestmark = pytest.mark.gpu


class PairGather:
    """all_gather for `world` managers in as many threads: every rank's buffer, concatenated rank-major."""

    def __init__(self, world):
        self.bufs = [None] * world
        self.barrier = threading.Barrier(world)
        self.out = None

    def rank(self, r):
        def all_gather(ptr, nbytes):
            self.bufs[r] = (ptr, nbytes)
            if self.barrier.wait() == 0:
                self.out = gather(self.bufs)
            self.barrier.wait()
            return self.out
        return all_gather


def placer(topo, **kw):
    e = TopoPlacer(device=0, **kw)
    e.set_topology(topo.row_ptr, topo.col_idx, topo.edge_w, topo.free, topo.domain, topo.domain_owner)
    return e


def key(p):
    return p.status, dict(p.nodes), p.domain, {k: list(v) for k, v in p.alternates.items()}


@pytest.mark.parametrize("committed", [False, True])
def test_world2_managers_give_the_world1_hints_and_alternates(committed):
    import bench
    topo = synth.make_topology(3000, seed=1)
    rbgs = bench.to_plugin(bench.fleet_spec("mooncake", 48, 3000, 0))
    e1 = placer(topo)
    ref = B200TopoPodGroupManager(e1, alternates=4).reconcile_pod_groups(rbgs, committed=committed)
    e1.close()
    assert any(p.alternates for p in ref)
    engs = [placer(topo, rank=r, world=2) for r in range(2)]
    pg = PairGather(2)
    mgrs = [B200TopoPodGroupManager(e, alternates=4, all_gather=pg.rank(r)) for r, e in enumerate(engs)]
    got, errs = [None, None], []

    def run(r):
        try:
            got[r] = mgrs[r].reconcile_pod_groups(rbgs, committed=committed)
        except BaseException as ex:   # reported below; a failed rank must not leave the other waiting
            errs.append(ex)
            pg.barrier.abort()
    ts = [threading.Thread(target=run, args=(r,)) for r in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    for e in engs:
        e.close()
    assert not errs, errs
    for r in range(2):
        assert [key(p) for p in got[r]] == [key(p) for p in ref], r

