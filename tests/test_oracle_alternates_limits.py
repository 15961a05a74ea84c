"""CPU: every designed case of tests/test_gpu_alternates_limits.py still hits its edge — each precondition asserted on
the oracles alone (tests/alternates_limits_cases.py), so a change to a generator or an oracle that moves a case off
its edge fails here without a GPU."""
import resource

import numpy as np
import pytest

import alternates_limits_cases as al


@pytest.mark.parametrize("own", al.OWN)
@pytest.mark.parametrize("kind", al.MERGE_KINDS)
def test_merge_cases(kind, own):
    topo, gblob, info = al.merge_case(kind, own)
    assert al.layout_holds(kind, al.layout(kind)[1])
    al.merge_pre(kind, own, topo, gblob, info)


@pytest.mark.parametrize("kind", al.MERGE_KINDS)
def test_colocated_merge_cases(kind):
    for own in ("rank0", "full"):
        topo, gblob, _ = al.merge_case(kind, own)
        for lv1 in (np.zeros(topo.n, np.int32), al.warp_of(np.arange(topo.n)).astype(np.int32) % 2):
            al.coloc_pre(topo, gblob, [(2, 1)], [topo.domain, lv1])


def test_job_ties_zero_row_and_count_cases():
    for demand in (0, 1):
        al.stack_pre(demand, *al.stack_case(demand))
    al.ties_pre(*al.ties_case())
    al.zero_row_pre(*al.zero_row_case())
    for F in range(9):
        al.count_pre(F, *al.count_case(F))


@pytest.mark.parametrize("n", al.BITMAP_NS)
def test_room_bitmap_cases(n):
    assert n % 4 != 0 and n > 64
    for pattern in (0, 1):
        al.bitmap_pre(*al.bitmap_case(n, pattern))
    topo, gblob, _ = al.bitmap_case(n, 0, level=1)
    al.level_bitmap_pre(topo, gblob, al.level_bitmap_levels(n))


def test_placement_list_case():
    al.many_used_pre(*al.many_used_case())


def test_chunk_case():
    topo, gblob = al.chunk_case()
    a, s, _ = al.committed_plain(topo, gblob)
    chunks, straddle = al.chunk_pre(topo, gblob, a, s)
    assert len(chunks) == 3 and straddle
    assert al.chunk_removed(topo, gblob, a, chunks)
    print(f"chunk case: peak host RSS {resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1024:.0f} MiB")


def test_eight_levels_case():
    al.eight_levels_pre(*al.eight_levels_case())


@pytest.mark.parametrize("i", range(len(al.EXACT)))
def test_exactness_cases(i):
    al.exact_pre(i, *al.exact_case(i))
