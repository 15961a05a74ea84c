"""Oracle of node eligibility in committed batches (rbgtopo_place_groups_eligible_committed[_ranked], DESIGN.md §3.20;
test infrastructure).

§3.20 adds §3.19's class term to every row of every round of the committed leader-worker loop.  So the oracle reuses
eligible_oracle.masked_rows (each row masked before lw_oracle.place_wave sees it) around the committed oracles and
restates no loop:
  * lw_committed_oracle.run_lw_committed (level 0, map or occupancy mode);
  * lw_committed_levels_oracle.run_lw_committed_levels[_ranked] (levels, RBGTOPO_CFG_LW_COMMIT_LEVELS);
  * lw_committed_alternates_oracle.run_lw_committed_ranked (level 0, ranked).
The ranked oracles keep the rows where run_group hands them to place_wave, so the mask has to sit inside that
row-keeping wrapper: their inner run is wrapped for the duration of the call, the way eligible_oracle.run_eligible_ranked
wraps lw_oracle.run_lw, and the rows they keep (and rank) are the masked ones."""
from __future__ import annotations

import contextlib

import lw_committed_alternates_oracle as lca
import lw_committed_levels_oracle as lclo
import lw_committed_oracle as lco
from eligible_oracle import default_role_pods, masked_rows


def _rp(gblob, role_pods):
    return default_role_pods(gblob) if role_pods is None else role_pods


@contextlib.contextmanager
def _masked_inner(module, name, gblob, rp, role_admit, node_class):
    """module.name runs inside masked_rows while the block lasts."""
    inner = getattr(module, name)

    def run(*a, **k):
        with masked_rows(gblob, rp, role_admit, node_class):
            return inner(*a, **k)

    setattr(module, name, run)
    try:
        yield
    finally:
        setattr(module, name, inner)


def run_eligible_committed(topo, gblob, role_pods, role_admit, node_class, **kw):
    """(assign, status, domain) of rbgtopo_place_groups_eligible_committed at level 0; role_pods None = (1, -1) per
    role; kw: as lw_committed_oracle.run_lw_committed (level_domain, owner0 for occupancy mode, limit)."""
    rp = _rp(gblob, role_pods)
    with masked_rows(gblob, rp, role_admit, node_class):
        return lco.run_lw_committed(topo, gblob, rp, **kw)


def run_eligible_committed_levels(topo, gblob, role_pods, role_admit, node_class, level_domain, owner, n_domains,
                                  **kw):
    """(assign, status, domain) at exclusive levels; arguments as lw_committed_levels_oracle.run_lw_committed_levels."""
    rp = _rp(gblob, role_pods)
    with masked_rows(gblob, rp, role_admit, node_class):
        return lclo.run_lw_committed_levels(topo, gblob, rp, level_domain, owner, n_domains, **kw)


def run_eligible_committed_ranked(topo, gblob, role_pods, role_admit, node_class, n_alt: int, **kw):
    """The six outputs of the ranked call at level 0 (assign, status, domain, score, alt_node, alt_score); kw: as
    lw_committed_alternates_oracle.run_lw_committed_ranked."""
    rp = _rp(gblob, role_pods)
    with _masked_inner(lco, "run_lw_committed", gblob, rp, role_admit, node_class):
        return lca.run_lw_committed_ranked(topo, gblob, rp, n_alt, **kw)


def run_eligible_committed_levels_ranked(topo, gblob, role_pods, role_admit, node_class, n_alt: int, level_domain,
                                         owner, n_domains):
    """The six outputs of the ranked call at exclusive levels."""
    rp = _rp(gblob, role_pods)
    with _masked_inner(lclo, "run_lw_committed_levels", gblob, rp, role_admit, node_class):
        return lclo.run_lw_committed_levels_ranked(topo, gblob, rp, n_alt, level_domain, owner, n_domains)
