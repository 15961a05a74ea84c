"""CPU: committed batches carry level hints when the placer places them (DESIGN.md §3.8 / §3.9): the GROUPS blob of a
committed reconcile holds every group with its key's index at word +10 when the placer has `places_committed_levels`,
and a placer that places levels but not committed levels keeps withholding those hints."""
from rbg_b200.plugin import RBGTOPO_NO_HINT, B200TopoPodGroupManager
from test_plugin_levels import KEYS, LevelsPlacer, groups


class CommittedLevelsPlacer(LevelsPlacer):
    places_committed_levels = True


def test_committed_blob_carries_the_key_index():
    pl = CommittedLevelsPlacer()
    mgr = B200TopoPodGroupManager(pl, exclusive_keys=KEYS)
    out = mgr.reconcile_pod_groups(groups(), committed=True)
    assert [p.status for p in out] == [1, 1, 1, 1, RBGTOPO_NO_HINT]   # "example.com/rack" is not configured
    gb = pl.blobs[-1]
    assert [(int(gb[8 + 12 * g]), int(gb[8 + 12 * g + 10])) for g in range(int(gb[2]))] == [(1, 0), (2, 1), (3, 2),
                                                                                            (4, 0)]
    assert set(mgr.no_hint) == {("ns", "e")}


def test_without_the_capability_committed_hints_are_withheld():
    pl = LevelsPlacer()
    assert not hasattr(pl, "places_committed_levels")
    mgr = B200TopoPodGroupManager(pl, exclusive_keys=KEYS)
    out = mgr.reconcile_pod_groups(groups(), committed=True)
    assert [p.status for p in out] == [1, RBGTOPO_NO_HINT, RBGTOPO_NO_HINT, 1, RBGTOPO_NO_HINT]
    gb = pl.blobs[-1]
    assert [int(gb[8 + 12 * g + 10]) for g in range(int(gb[2]))] == [0, 0]


def test_snapshot_batches_are_unchanged_by_the_capability():
    a, b = CommittedLevelsPlacer(), LevelsPlacer()
    for pl in (a, b):
        B200TopoPodGroupManager(pl, exclusive_keys=KEYS).reconcile_pod_groups(groups())
    assert (a.blobs[-1] == b.blobs[-1]).all()
