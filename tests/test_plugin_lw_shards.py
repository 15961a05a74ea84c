"""GPU: the plugin with leader-worker groups on a world = 2 pair of placers created with lw_shards=True (DESIGN.md
§3.18; two contexts on one device, each behind its own B200TopoPodGroupManager with leader_worker=True, reconciling
from two threads).  The managers' all-gather concatenates the two exchange buffers on the device.  Hints and
alternates, keyed by pod name, must equal those of the world = 1 plugin for snapshot and committed batches, with and
without alternates."""
import threading

import pytest

from rbg_b200 import synth
from rbg_b200.engine import TopoPlacer
from rbg_b200.plugin import GANG_SCHEDULING_KEY, B200TopoPodGroupManager
from test_plugin_lw import lws_group, plain_group
from test_plugin_shard_alternates import PairGather, key, placer

pytestmark = pytest.mark.gpu


def fleet():
    gang = {GANG_SCHEDULING_KEY: "true"}
    return [lws_group("a", 1, lws=4), plain_group("b", 2), lws_group("c", 3, colocate="any", lws=2),
            lws_group("d", 4, lws=8, ann=gang), lws_group("e", 1, lws=2), plain_group("f", 5)]


@pytest.mark.parametrize("committed", [False, True])
@pytest.mark.parametrize("alternates", [0, 4])
def test_world2_managers_give_the_world1_hints_and_alternates(committed, alternates):
    topo = synth.make_topology(1000, seed=4, tiers=2, max_free=3)
    topo.domain_owner[:] = -1
    rbgs = fleet()
    e1 = placer(topo)
    ref = B200TopoPodGroupManager(e1, alternates=alternates, leader_worker=True).reconcile_pod_groups(
        rbgs, committed=committed)
    e1.close()
    assert any(len(p.nodes) > 3 for p in ref) and any("a-decode-0-3" in p.nodes for p in ref)
    if alternates:
        assert any(p.alternates for p in ref)
    engs = [placer(topo, rank=r, world=2, lw_shards=True) for r in range(2)]
    pg = PairGather(2)
    mgrs = [B200TopoPodGroupManager(e, alternates=alternates, leader_worker=True, all_gather=pg.rank(r))
            for r, e in enumerate(engs)]
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
        assert not mgrs[r].no_hint, mgrs[r].no_hint
        assert [key(p) for p in got[r]] == [key(p) for p in ref], r
