"""Oracle of node eligibility (rbgtopo_place_groups_eligible[_ranked], DESIGN.md §3.19; test infrastructure).

§3.19 adds one feasibility term to the leader-worker loop: role rho may not use node n when bit class[n] of its mask
admit_rho is clear, and its dense-row entry there is -inf.  So the oracle masks every row before
lw_oracle.place_wave sees it, by wrapping that function the way lw_alternates_oracle wraps it, and lets
lw_oracle.run_lw and lw_alternates_oracle.run_lw_ranked do everything else; neither loop is restated.  The ranked form
wraps lw_oracle.run_lw for the duration of the call, so the mask is applied inside run_lw_rows' own wrapper: the rows it
keeps (and ranks) are the masked ones."""
from __future__ import annotations

import contextlib

import numpy as np

import lw_alternates_oracle as la
import lw_oracle as lw

ALL = (1 << 64) - 1


def admits(mask: int, node_class) -> np.ndarray:
    """Boolean vector: bit node_class[n] of mask is set."""
    cls = np.asarray(node_class, dtype=np.uint64)
    return ((np.uint64(int(mask) & ALL) >> cls) & np.uint64(1)).astype(bool)


def default_role_pods(gblob) -> np.ndarray:
    """role_pods == NULL: (S, C) = (1, -1) for every role."""
    return lw.role_pods_for(gblob, lambda g, r: (1, -1))


@contextlib.contextmanager
def masked_rows(gblob, role_pods, role_admit, node_class):
    """Inside the block lw_oracle.place_wave receives each row with -inf where its role does not admit the node."""
    masks = [int(m) for m in np.asarray(role_admit, dtype=np.uint64).reshape(-1)]
    groups = la.groups_of(gblob, role_pods)
    r0 = np.concatenate([[0], np.cumsum([X.q for X in groups])]).astype(int)
    first_pod = {X.pod0: g for g, X in enumerate(groups) if X.n_pods}
    inner = lw.place_wave

    def mask(G, w, wave_rows, *args, **kw):
        g = first_pod[G.pod0]
        rows = []
        for p, row in enumerate(wave_rows):
            ok = admits(masks[r0[g] + G.waves[w][p][0]], node_class)
            rows.append(np.where(ok, row, np.float32(-np.inf)).astype(np.float32))
        return inner(G, w, rows, *args, **kw)

    lw.place_wave = mask
    try:
        yield
    finally:
        lw.place_wave = inner


def run_eligible(topo, gblob, role_pods, role_admit, node_class, **kw):
    """(assign, status, domain) of rbgtopo_place_groups_eligible; role_pods None = (1, -1) per role.  kw: as
    lw_oracle.run_lw."""
    rp = default_role_pods(gblob) if role_pods is None else role_pods
    with masked_rows(gblob, rp, role_admit, node_class):
        return lw.run_lw(topo, gblob, rp, **kw)


def run_eligible_ranked(topo, gblob, role_pods, role_admit, node_class, n_alt: int, **kw):
    """The six outputs of rbgtopo_place_groups_eligible_ranked; kw: as lw_alternates_oracle.run_lw_ranked."""
    rp = default_role_pods(gblob) if role_pods is None else role_pods
    inner_run = lw.run_lw

    def run(*a, **k):
        with masked_rows(gblob, rp, role_admit, node_class):
            return inner_run(*a, **k)

    lw.run_lw = run
    try:
        return la.run_lw_ranked(topo, gblob, rp, n_alt, **kw)
    finally:
        lw.run_lw = inner_run


def full_masks(gblob) -> np.ndarray:
    """Every role admits every class."""
    gb = np.asarray(gblob, dtype=np.int64)
    q = sum(int(gb[lw.HDR + lw.GW * g + 3]) for g in range(int(gb[2])))
    return np.full(q, ALL, dtype=np.uint64)
