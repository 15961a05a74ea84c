"""Fixtures of the batch-reuse tests (test infrastructure).

Every placement entry point runs on a batch taken from the context's pool, and a single-threaded caller always gets the
pool's first free batch: one entry point after another reuses the same device and pinned buffers, which only ever grow
and are never cleared.  A `World` is one snapshot (topology, installed partitions, context flags) with a *small* and a
*large* fixture per family of entry points, all on that one topology, so that any call can follow any other on one
context:

  steps   step-level BLOBs (score_assign, stage / run_staged / fetch), steps_gen's kinds;
  groups  GROUPS blobs (place_groups direct and staged, _committed[_ranked], _ranked): the lw fleet's groups, the large
          fixture with two 16-role groups on top (8-role waves, 32-replica waves, roles split across waves);
  lw      GROUPS blobs with (S, C) per role (_lw[_ranked], _lw_committed[_ranked]).

The small fixture is not a prefix of the large one (other groups, other order, fewer pods per replica), so what a call
leaves in the pool's buffers differs from what the next call writes there: tests/test_reuse_cases.py asserts that on
the oracles.  `growth_steps` sits either side of DevBuf's growth rule, `failing` holds calls that fail after their blob
was uploaded."""
from __future__ import annotations

import dataclasses
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np

import groups_gen as gg
import lw_commit_gen as lg
import lw_commit_levels_gen as lvg
import steps_gen as sg
from rbg_b200 import synth
from rbg_b200.blob import STEP_EXCLUSIVE, STEP_GANG, Group

# every entry point of the pool (the set K)
KINDS = ("score_assign", "steps", "direct", "staged", "committed", "committed_ranked", "ranked", "lw", "lw_ranked",
         "lw_committed", "lw_committed_ranked")
FAMILY = {"score_assign": "steps", "steps": "steps", "direct": "groups", "staged": "groups", "committed": "groups",
          "committed_ranked": "groups", "ranked": "groups", "lw": "lw", "lw_ranked": "lw", "lw_committed": "lw",
          "lw_committed_ranked": "lw"}
SIZES = ("small", "large")
N_ALT = 8
SMALL_PICK = (11, 4, 7)        # groups of the small fixtures, in this order: not a prefix of the large ones


def grow(n: int) -> int:
    """DevBuf::reserve's capacity after a request of n elements."""
    return n + n // 4 + 64


def slab_stride(n: int) -> int:
    """Row stride of the dense matrix on one rank with the default chunk (rbgtopo.cu, slab geometry)."""
    tcfg = 2048
    lc = max(1, (n + tcfg - 1) // tcfg)
    chunk = min(2048, max(128, -(-((n + lc - 1) // lc) // 128) * 128))
    return -(-(lc * chunk) // 32) * 32


@dataclass
class Fixture:
    family: str
    blob: np.ndarray
    groups: List = field(default_factory=list)   # Group (groups / lw) or Step (steps) records of the blob
    rp: Optional[np.ndarray] = None               # lw: (S, C) per role


@dataclass
class World:
    name: str
    topo: synth.Topology
    lv: Optional[np.ndarray] = None    # [n_levels + 1][n] (row 0 = domain): partitions installed on the context
    nd: Optional[List[int]] = None
    occ: Optional[np.ndarray] = None
    flags: Dict[str, bool] = field(default_factory=dict)   # TopoPlacer keyword flags
    fx: Dict[Tuple[str, str], Fixture] = field(default_factory=dict)   # (family, size) -> fixture

    def fixture(self, kind: str, size: str) -> Fixture:
        return self.fx[(FAMILY[kind], size)]

    def owner0(self) -> np.ndarray:
        """The level-0 owner the selection reads: derived from the records once partitions are installed."""
        if self.lv is None:
            return self.topo.domain_owner
        import levels_oracle as lo
        return lo.derive_level_owner(self.lv, self.occ)[0]


def _steps(topo, seed: int, n_steps: int, kinds=sg.KINDS) -> List:
    """steps_gen steps on `topo` (a copy takes the owner changes some kinds make: the blob stays valid on topo)."""
    import topo_gen as tg
    t = tg.copy_topo(topo)
    t.domain_owner = t.domain_owner.copy()
    deg = np.diff(t.row_ptr)
    hubs = [int(np.argmax(deg))]
    iso = np.nonzero(deg == 0)[0].tolist()
    rng = np.random.default_rng(seed)
    limit = sg.amax_limit(t)
    return [sg._step(rng, kinds[(s + seed) % len(kinds)], t, hubs, iso, limit) for s in range(n_steps)]


def _wide(topo, seed: int, gids) -> List[Group]:
    """16-role groups of groups_gen on `topo`: a level of 10 roles (a wave of 8 role rows), a level that sums past 32
    replicas (a wave of exactly 32, a role split across waves); exclusive, the first one a gang."""
    rng = np.random.default_rng(seed)
    row_w = gg.wsum_max(topo)
    out = []
    for i, gid in enumerate(gids):
        roles = gg._wide(rng, int(topo.free.max()) + 1)
        g = Group(gid=gid, roles=roles, pair=gg._pair(rng, len(roles), zero_row=i == 0),
                  anchors=[(int(rng.integers(0, topo.n)), int(rng.integers(0, len(roles))), 2)],
                  flags=STEP_EXCLUSIVE | (STEP_GANG if i == 0 else 0))
        while not gg.exact_ok(g, row_w):
            p = np.asarray(g.pair)
            p[np.unravel_index(int(np.argmax(p)), p.shape)] -= 1
            g.pair = p.tolist()
        out.append(g)
    return out


def _rp(rps) -> np.ndarray:
    return np.asarray([sc for g in rps for sc in g], dtype=np.int32).reshape(-1, 2)


def _fill(w: World, groups, rps, seed: int) -> World:
    """The three families' fixtures of a world from one fleet's groups and (S, C)."""
    small = [groups[k] for k in SMALL_PICK]
    small_rp = [[(max(1, S // 2), C) for S, C in rps[k]] for k in SMALL_PICK]   # fewer pods per replica
    wide = _wide(w.topo, seed + 50, gids=(groups[0].gid, 77))
    w.fx[("groups", "large")] = Fixture("groups", lg.build(list(groups) + wide), list(groups) + wide)
    w.fx[("groups", "small")] = Fixture("groups", lg.build(small), small)
    w.fx[("lw", "large")] = Fixture("lw", lg.build(list(groups)), list(groups), _rp(rps))
    w.fx[("lw", "small")] = Fixture("lw", lg.build(small), small, _rp(small_rp))
    big = _steps(w.topo, seed + 100, 17)
    few = _steps(w.topo, seed + 200, 3)
    w.fx[("steps", "large")] = Fixture("steps", sg.build(big), big)
    w.fx[("steps", "small")] = Fixture("steps", sg.build(few), few)
    return w


def plain_world(seed: int = 4, n: int = 513) -> World:
    """A level-0 context: lw_commit_gen's scarce fleet of 14 groups (exclusive, gang, fixed domains, shared gids)."""
    f = lg.fleet(seed, n, n_groups=14, scarce=True)
    return _fill(World(f"plain{n}", f.topo), f.groups, f.rp, seed)


def level_world(seed: int = 4, n: int = 513) -> World:
    """The flags = 7 context with levels 1..3 installed (lw_commit_levels_gen): groups at exclusive levels 0..3,
    co-location levels -1..3, records of the fleet's gids and of one outsider."""
    f = lvg.fleet(seed, n, n_groups=14, scarce=True, kind="mixed")
    w = World(f"levels{n}", f.topo, f.lv, f.nd, f.occ, dict(lw_committed_levels=True))
    w = _fill(w, f.groups, f.rp, seed)
    for size in SIZES:   # the small fixtures must reach a level >= 1
        assert any(g.level > 0 for g in w.fx[("groups", size)].groups), size
    return w


def level0_world(seed: int = 4, n: int = 513) -> World:
    """level_world's snapshot and partitions on a context WITHOUT the level flags, with the same fleet at level 0:
    a group at a level >= 1 answers RBGTOPO_ELIMIT here."""
    lw = level_world(seed, n)
    f = lg.fleet(seed, n, n_groups=14, scarce=True, levels=True)   # the groups lvg.fleet moved to levels
    w = World(f"level0_{n}", lw.topo, lw.lv, lw.nd, lw.occ, {})
    return _fill(w, f.groups, f.rp, seed)


def growth_steps(w: World):
    """(A, B fitting, B growing) step blobs on w: A has 8 role rows (one 8-role step), so the dense matrix is reserved
    for grow(8 * stride) floats; B fitting has 10 role rows, which fit that capacity (its rows 0..7 hold A's rows, its
    rows 8..9 the reservation's unwritten tail), B growing has 11, one row past it, which reallocates."""
    wide = _steps(w.topo, 301, 3, kinds=("wide",))
    single = _steps(w.topo, 302, 3, kinds=("single",))
    a = sg.build(wide[:1])
    fit = sg.build(wide[1:2] + single[:2])
    grows = sg.build(wide[2:3] + single[:3])
    return a, fit, grows


# ---- calls that fail after their blob was pre-uploaded

FAILING_NAMES = ("einval_score_assign", "einval_stage", "einval_direct", "einval_stage_groups", "einval_committed",
                 "einval_ranked", "einval_lw_committed_ranked", "einexact_lw", "einexact_lw_ranked",
                 "einexact_lw_committed", "einexact_ranked", "einexact_committed_ranked")
ELIMIT_NAMES = ("elimit_direct", "elimit_stage_groups", "elimit_committed", "elimit_ranked", "elimit_lw",
                "elimit_lw_committed_ranked")

def bad_word(blob: np.ndarray) -> np.ndarray:
    """The blob with its last word (an anchor count, a consumed record's capacity or a pair weight: the body's tail)
    set to -5: EINVAL, found only when validation reaches the last record."""
    b = np.array(blob, dtype=np.int32, copy=True)
    b[-1] = -5
    return b


def at_level(groups, k: int = 0) -> np.ndarray:
    """The groups with group k moved to exclusive level 1 (ELIMIT on a context without RBGTOPO_CFG_LEVEL_PLACEMENT)."""
    gs = list(groups)
    gs[k] = dataclasses.replace(gs[k], level=1, fixed_domain=-1, flags=gs[k].flags | STEP_EXCLUSIVE)
    return lg.build(gs)


def lw_inexact(topo):
    """test_gpu_lw_limits' first enumerated case on `topo`: the anchor count at the exactness bound of the pod waves
    (every mix of unplaced earlier pods), where place_groups_lw / _lw_ranked / _lw_committed answer EINEXACT."""
    from test_gpu_lw_limits import EXACT_CASES, enumerated_bound, exact_group
    pair, S, pend, gang = EXACT_CASES[0]
    roles, full = exact_group(pair, pend)
    B = enumerated_bound(roles[:-1], [r[:-1] for r in full[:-1]], list(S), gang)
    row_w = gg.wsum_max(topo) + 8000
    c_at = ((1 << 24) + row_w - 1) // row_w - max(B)
    blob = lg.build([Group(gid=1, roles=roles, pair=full, anchors=[(7, len(pend), c_at)],
                           flags=STEP_GANG if gang else 0)])
    return blob, np.asarray([(s, -1) for s in S] + [(1, -1)], dtype=np.int32)


def ranked_inexact(topo):
    """alternates_limits_cases' second exactness case on `topo`: the anchor count at the bound of the ranking, where
    place_groups_ranked and _committed_ranked answer EINEXACT."""
    import alternates_limits_cases as alc
    from test_gpu_lw_limits import exact_group
    pair, pend = alc.EXACT[1]
    roles, full = exact_group(pair, pend)
    B = alc.enumerated_bound(roles[:-1], [r[:-1] for r in full[:-1]], False)
    c_at = alc.anchor_limit(topo) - max(B)
    return lg.build([Group(gid=1, roles=roles, pair=full, anchors=[(7, len(pend), c_at)])])


def failing(w: World):
    """(name, entry point, arguments, expected code) of the failing calls on a level-0 world."""
    gb = w.fx[("groups", "large")].blob
    lf = w.fx[("lw", "large")]
    sb = w.fx[("steps", "large")].blob
    out = [("einval_score_assign", "score_assign", (bad_word(sb),), -1),
           ("einval_stage", "stage", (bad_word(sb),), -1),
           ("einval_direct", "place_groups", (bad_word(gb),), -1),
           ("einval_stage_groups", "stage_groups", (bad_word(gb),), -1),
           ("einval_committed", "place_groups_committed", (bad_word(gb),), -1),
           ("einval_ranked", "place_groups_ranked", (bad_word(gb), N_ALT), -1),
           ("einval_lw_committed_ranked", "place_groups_lw_committed_ranked", (bad_word(lf.blob), lf.rp, N_ALT), -1)]
    lb, lrp = lw_inexact(w.topo)
    out += [("einexact_lw", "place_groups_lw", (lb, lrp), -4),
            ("einexact_lw_ranked", "place_groups_lw_ranked", (lb, lrp, N_ALT), -4),
            ("einexact_lw_committed", "place_groups_lw_committed", (lb, lrp), -4)]
    rb = ranked_inexact(w.topo)
    out += [("einexact_ranked", "place_groups_ranked", (rb, N_ALT), -4),
            ("einexact_committed_ranked", "place_groups_committed_ranked", (rb, N_ALT), -4)]
    return out


def failing_levels(w: World):
    """ELIMIT on level0_world: a large blob with its first group at level 1, through every GROUPS entry point."""
    gs = w.fx[("groups", "large")].groups
    lf = w.fx[("lw", "large")]
    gb, lb = at_level(gs), at_level(lf.groups)
    return [("elimit_direct", "place_groups", (gb,), -6),
            ("elimit_stage_groups", "stage_groups", (gb,), -6),
            ("elimit_committed", "place_groups_committed", (gb,), -6),
            ("elimit_ranked", "place_groups_ranked", (gb, N_ALT), -6),
            ("elimit_lw", "place_groups_lw", (lb, lf.rp), -6),
            ("elimit_lw_committed_ranked", "place_groups_lw_committed_ranked", (lb, lf.rp, N_ALT), -6)]


# ---- topology changes: N = 4 097 -> 129 -> 65 537 -> 4 097
TOPO_SEQUENCE = (4097, 129, 65537, 4097)
TOPO_SEED = 6
