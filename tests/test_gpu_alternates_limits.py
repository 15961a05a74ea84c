"""GPU: ranked alternates at their limits (rbgtopo_place_groups_ranked, DESIGN.md §3.10, and
rbgtopo_place_groups_committed_ranked, §3.14) bit for bit against tests/alternates_oracle.py and
tests/committed_alternates_oracle.py, with assign / status / domain (/ rounds) equal to the unranked calls', plus
invariants read from the outputs alone: alternates strictly descending by key(score, node), never the replica's own
node, unfilled slots (-1 / -inf) only after filled ones; for a committed batch, moving one replica to one of its
alternates keeps that node within free over the whole batch and breaks no anti-affinity term of the records or of the
batch's placed pods.

Cases (tests/alternates_limits_cases.py; each asserts its precondition on the oracle first): the top-list merge with
the nine winners in thread 0's stride set, in one warp, one per warp, in warp 7, each with the replica's node at row
rank 0, at row rank 8 and without room (a node that keeps room always heads its candidates: the greedy took the best
node with room, and room only shrinks afterwards); a 32-replica job; ties; a row of +0.0; exactly n_alt, n_alt + 1
and fewer candidates at every n_alt; the co-located leader-worker form on the same layouts; the room bitmap at nodes
0, 31, 32, 63 and n - 1 of ragged N, a placement list longer than the 256 threads that mark it, a demand-0 role, an
exclusive group at level 1; the committed replay in three chunks at 1 638 400 nodes; a committed batch at all eight
exclusive levels; the exactness bound of the ranking against an enumeration of the worst mix of unplaced replicas."""
import ctypes as C
import resource

import numpy as np
import pytest

import alternates_limits_cases as al
import committed_alternates_oracle as cao
import committed_levels_oracle as clo
import levels_oracle as lo
from oracle import wave_loop
from rbg_b200 import _lib
from rbg_b200.engine import _p
from test_gpu_lw_limits import engine, oracle_lw, raw, same as lw_same

pytestmark = pytest.mark.gpu

EINEXACT = -4
SENT = 0x5A5A5A5A


def bits(x):
    x = np.asarray(x)
    return x.view(np.uint32) if x.dtype == np.float32 else x


def equal(got, exp, F, what):
    """got / exp: (assign, status, domain, score, alt_node, alt_score); exp ranked at n_alt >= F."""
    exp = tuple(exp[:4]) + (np.asarray(exp[4])[:, :F], np.asarray(exp[5])[:, :F])
    for i, (x, y) in enumerate(zip(got, exp)):
        assert np.array_equal(bits(x), bits(y)), (what, F, i, np.nonzero(bits(x) != bits(y))[0][:8])


def invariants(a, sc, an, asc):
    for r in range(len(a)):
        k = int((an[r] >= 0).sum())
        assert (an[r][:k] >= 0).all() and (an[r][k:] == -1).all(), (r, an[r])
        assert np.isfinite(asc[r][:k]).all() and np.isneginf(asc[r][k:]).all(), (r, asc[r])
        if a[r] < 0:
            assert k == 0 and np.isneginf(sc[r]), r
            continue
        assert a[r] not in an[r][:k], (r, a[r], an[r])
        s, m = asc[r][:k], an[r][:k]
        assert ((s[:-1] > s[1:]) | ((s[:-1] == s[1:]) & (m[:-1] < m[1:]))).all(), (r, m, s)


def check_ranked(eng, topo, gblob, F, exp):
    got = eng.place_groups_ranked(gblob, F)
    for x, y in zip(got[:3], eng.place_groups(gblob)):
        assert np.array_equal(x, y)
    equal(got, exp, F, "place_groups_ranked")
    invariants(got[0], got[3], got[4], got[5])
    return got


def batch_room(topo, gblob, a, an):
    """Every alternate x of replica r: free[x] - (demand the whole batch placed on x) >= demand of r."""
    rooms = al.room_after(topo, gblob, a, committed=True)
    i = 0
    for room, dem in rooms:
        for d in dem:
            x = an[i][an[i] >= 0]
            assert (room[x] >= d).all(), (i, x, room[x], d)
            i += 1


def alt_violations(lv, occ, gblob, a, s, an):
    """Alternates of participating replicas that break an anti-affinity term of the records or of a placed pod."""
    groups = wave_loop.groups_from_blob(gblob)
    levels = clo.group_levels(gblob)
    pods, reps, i = [tuple(int(v) for v in x) for x in np.asarray(occ).reshape(-1, 3)], [], 0
    for g, G in enumerate(groups):
        st = wave_loop.GroupState(G)
        for ri in st.order:
            for _ in range(st.pending[ri]):
                if G.exclusive and G.roles[ri].exclusive and a[i] >= 0 and s[g] != 2:
                    pods.append((int(a[i]), G.gid, levels[g]))
                    reps.append((i, G.gid, levels[g]))
                i += 1
    occ_all = np.array(pods, np.int64).reshape(-1, 3)
    return [(r, int(x)) for r, gid, L in reps for x in an[r] if x >= 0
            and lo.violates(lv, al.KEYS[:len(lv)], occ_all, gid, L, int(x))]


def check_committed(eng, topo, gblob, F, exp, lv=None, occ=None):
    got = eng.place_groups_committed_ranked(gblob, F)
    a, s, d, rounds, sc, an, asc = got
    plain = eng.place_groups_committed(gblob)
    assert all(np.array_equal(x, y) for x, y in zip(plain[:3], (a, s, d))) and plain[3] == rounds
    equal((a, s, d, sc, an, asc), exp, F, "place_groups_committed_ranked")
    invariants(a, sc, an, asc)
    batch_room(topo, gblob, a, an)
    if lv is not None:
        assert alt_violations(lv, occ, gblob, a, s, an) == []
    return got


def committed_oracle(topo, gblob, F=8, **kw):
    return cao.run_fleet_committed_ranked(topo, wave_loop.groups_from_blob(gblob), F, fast=True, **kw)


# ---- 1. the top-list merge

@pytest.mark.parametrize("own", al.OWN)
@pytest.mark.parametrize("kind", al.MERGE_KINDS)
def test_merge_edges(kind, own):
    topo, gblob, info = al.merge_case(kind, own)
    exp = al.merge_pre(kind, own, topo, gblob, info)
    eng = engine(topo)
    try:
        for F in (8, 3):
            check_ranked(eng, topo, gblob, F, exp)
        check_committed(eng, topo, gblob, 8, committed_oracle(topo, gblob))
    finally:
        eng.close()


@pytest.mark.parametrize("demand", [0, 1])
def test_one_job_of_thirty_two_replicas(demand):
    topo, gblob = al.stack_case(demand)
    exp = al.stack_pre(demand, topo, gblob)
    eng = engine(topo)
    try:
        check_ranked(eng, topo, gblob, 8, exp)
        check_committed(eng, topo, gblob, 8, committed_oracle(topo, gblob))
    finally:
        eng.close()


def test_ties_over_more_than_nine_nodes_and_a_row_of_zeros():
    topo, gblob, nodes = al.ties_case()
    exp = al.ties_pre(topo, gblob, nodes)
    eng = engine(topo)
    try:
        check_ranked(eng, topo, gblob, 8, exp)
    finally:
        eng.close()
    topo, gblob = al.zero_row_case()
    exp = al.zero_row_pre(topo, gblob)
    eng = engine(topo)
    try:
        check_ranked(eng, topo, gblob, 8, exp)
        check_committed(eng, topo, gblob, 8, committed_oracle(topo, gblob))
    finally:
        eng.close()


@pytest.mark.parametrize("F", range(9))
def test_exactly_n_alt_one_more_and_fewer_candidates(F):
    topo, gblob = al.count_case(F)
    exp = al.count_pre(F, topo, gblob)
    eng = engine(topo)
    try:
        check_ranked(eng, topo, gblob, F, exp)
        check_committed(eng, topo, gblob, F, committed_oracle(topo, gblob))
    finally:
        eng.close()


@pytest.mark.parametrize("kind", al.MERGE_KINDS)
def test_colocated_pods_on_the_merge_layouts(kind):
    """place_groups_lw_ranked (k_alternates<true>): S = 2 pods co-located at level 1, a single domain (the row's
    whole layout) or the warps' parity (half of it), on the rank0 and full layouts."""
    for own in ("rank0", "full"):
        topo, gblob, _ = al.merge_case(kind, own)
        n = topo.n
        for lv1 in (np.zeros(n, np.int32), al.warp_of(np.arange(n)).astype(np.int32) % 2):
            lvl = [topo.domain, lv1]
            rp = np.array([(2, 1)], np.int32)
            exp = al.coloc_pre(topo, gblob, rp, lvl)
            eng = engine(topo, lvl)
            try:
                for F in (8, 1):
                    lw_same(eng.place_groups_lw_ranked(gblob, rp, F), exp, F)
            finally:
                eng.close()


# ---- 2. the room bitmap

@pytest.mark.parametrize("pattern", [0, 1])
@pytest.mark.parametrize("n", al.BITMAP_NS)
def test_room_bitmap_edges(n, pattern):
    topo, gblob, info = al.bitmap_case(n, pattern)
    exp = al.bitmap_pre(topo, gblob, info)
    eng = engine(topo)
    try:
        for F in (8, 2):
            check_ranked(eng, topo, gblob, F, exp)
        check_committed(eng, topo, gblob, 8, committed_oracle(topo, gblob))
    finally:
        eng.close()


def test_placement_list_longer_than_the_marking_threads():
    topo, gblob = al.many_used_case()
    exp = al.many_used_pre(topo, gblob)
    eng = engine(topo)
    try:
        check_ranked(eng, topo, gblob, 8, exp)
        check_committed(eng, topo, gblob, 8, committed_oracle(topo, gblob))
    finally:
        eng.close()


@pytest.mark.parametrize("n", al.BITMAP_NS)
def test_exclusive_group_at_level_one_at_ragged_n(n):
    """RBGTOPO_CFG_LEVEL_PLACEMENT: the participating roles' candidates test the level-1 domain vector, read with
    16-byte loads past n; place_groups_ranked against the leader-worker oracle with one pod per replica."""
    topo, gblob, _ = al.bitmap_case(n, 0, level=1)
    lvl = al.level_bitmap_levels(n)
    ones = np.array([(1, -1)] * 3, np.int32)
    exp = al.level_bitmap_pre(topo, gblob, lvl)
    eng = engine(topo, lvl, level_placement=True)
    try:
        for F in (8, 2):
            got = eng.place_groups_ranked(gblob, F)
            for x, y in zip(got[:3], eng.place_groups(gblob)):
                assert np.array_equal(x, y)
            lw_same(got, exp, F)
            invariants(got[0], got[3], got[4], got[5])
        lw_same(eng.place_groups_lw_ranked(gblob, ones, 8), exp, 8)
    finally:
        eng.close()


# ---- 3. the committed replay across chunks

def test_committed_replay_across_chunks():
    """1 638 400 nodes: slab_stride 1 638 400, so a replay chunk holds 163 rows; 351 rows make three.  Group 11's
    waves fall in two chunks with its empty wave at the boundary, a gang-failed group is skipped, and group 0 alone
    would have alternates that groups of later chunks take.  The launch count gives the chunks: 2 per chunk on top of
    place_groups_committed's 3 · rounds + 1."""
    topo, gblob = al.chunk_case()
    assert al.slab_stride(topo.n) == topo.n and al.REPLAY_FLOATS // topo.n == 163
    exp = committed_oracle(topo, gblob)
    chunks, straddle = al.chunk_pre(topo, gblob, exp[0], exp[1])
    assert len(chunks) == 3 and al.chunk_removed(topo, gblob, exp[0], chunks)
    eng = engine(topo)
    try:
        for F in (8, 1):
            got = check_committed(eng, topo, gblob, F, exp)
            eng.place_groups_committed_ranked(gblob, F)
            launches = eng.last_timing()["launches"]
            assert launches == 3 * got[3] + 1 + 2 * len(chunks), (launches, got[3], len(chunks))
    finally:
        eng.close()
    print(f"committed replay across chunks: peak host RSS "
          f"{resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1024:.0f} MiB")


# ---- 4. all eight levels

def test_committed_batch_at_all_eight_levels():
    topo, lv, nd, occ, base, gblob, picked = al.eight_levels_case()
    exp = al.eight_levels_pre(topo, lv, nd, occ, base, gblob, picked)
    eng = engine(topo, committed_levels=True)
    try:
        eng.set_exclusive_levels(lv[1:], occ, level_n_domains=nd[1:])
        for F in (1, 8):
            check_committed(eng, topo, gblob, F, exp, lv=lv, occ=occ)
    finally:
        eng.close()


# ---- 5. the exactness bound of the ranking

def raw_committed_ranked(eng, gblob, F=3):
    gb = np.ascontiguousarray(gblob, np.int32)
    P, ng = int(gb[4]), int(gb[2])
    outs = [np.full(P + 1, SENT, np.int32), np.full(ng + 1, SENT, np.int32), np.full(ng + 1, SENT, np.int32),
            np.full(P + 1, SENT, np.int32), np.full((P + 1) * F, SENT, np.int32), np.full((P + 1) * F, SENT, np.int32)]
    rounds = C.c_int32(9)
    f = lambda x: _p(x.view(np.float32), _lib.f32p)
    rc = eng.lib.rbgtopo_place_groups_committed_ranked(eng._h, _p(gb), len(gb), F, _p(outs[0]), _p(outs[1]),
                                                       _p(outs[2]), C.byref(rounds), f(outs[3]), _p(outs[4]),
                                                       f(outs[5]))
    return rc, all((x == SENT).all() for x in outs), rounds.value


@pytest.mark.parametrize("i", range(len(al.EXACT)))
def test_exactness_bound_of_the_ranking(i):
    """At the enumerated bound the committed-ranked call refuses with RBGTOPO_EINEXACT, outputs untouched, rounds 0;
    one anchor below it places and matches the oracle.  place_groups_ranked on the same blobs either matches its
    oracle or refuses before writing anything."""
    topo, blob, c_at, B = al.exact_case(i)
    al.exact_pre(i, topo, blob, c_at, B)
    eng = engine(topo)
    try:
        rc, untouched, rounds = raw_committed_ranked(eng, blob(c_at))
        assert rc == EINEXACT and untouched and rounds == 0, (rc, untouched, rounds, B, c_at)
        check_committed(eng, topo, blob(c_at - 1), 8, committed_oracle(topo, blob(c_at - 1)))
        for c in (c_at, c_at - 1):
            rc, untouched = raw(eng, "ranked", blob(c))
            if rc == 0:
                check_ranked(eng, topo, blob(c), 8, al.ranked(topo, blob(c)))
            else:
                assert rc == EINEXACT and untouched, (c, rc)
    finally:
        eng.close()
