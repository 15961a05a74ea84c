"""Object wrapper over one rbgtopo_ctx (C ABI of include/rbgtopo.h)."""
from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import numpy as np

from . import _lib
from .blob import blob_totals


def plan_steps(groups_blob, n_nodes: int = 4096, n_domains: int = 1) -> np.ndarray:
    """Host-only: the step geometry of the multi-wave plan rbgtopo_place_groups / _stage_groups
    compile from a GROUPS blob (rbgtopo_plan_describe).  One row of 8 ints per step, wave-major:
    group, wave, section offset, section end, first replica row, first role row, next step, i0."""
    lib = _lib.load()
    gb = np.ascontiguousarray(groups_blob, dtype=np.int32)
    ns, nw, pw = C.c_int32(), C.c_int32(), C.c_int64()
    i32 = _lib.i32p
    rc = lib.rbgtopo_plan_describe(gb.ctypes.data_as(i32), len(gb), n_nodes, n_domains, None, 0, None, 0,
                                   C.byref(ns), C.byref(nw), C.byref(pw))
    if rc != 0:
        raise RuntimeError(f"rbgtopo_plan_describe: {rc}")
    out = np.zeros(max(ns.value, 1) * 8, dtype=np.int32)
    rc = lib.rbgtopo_plan_describe(gb.ctypes.data_as(i32), len(gb), n_nodes, n_domains, None, 0,
                                   out.ctypes.data_as(i32), ns.value, C.byref(ns), C.byref(nw), C.byref(pw))
    if rc != 0:
        raise RuntimeError(f"rbgtopo_plan_describe: {rc}")
    return out[:ns.value * 8].reshape(-1, 8)


class RbgTopoError(RuntimeError):
    def __init__(self, code: int, text: str):
        super().__init__(f"rbgtopo error {code}: {text}")
        self.code = code


def _p(a: Optional[np.ndarray], typ=_lib.i32p):
    return None if a is None else a.ctypes.data_as(typ)


def _i32(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.int32)


class _DevBytes:
    """A device buffer the library owns, as a uint8 array for torch.as_tensor."""

    def __init__(self, ptr: int, nbytes: int):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 3,
                                         "strides": None}


class TopoPlacer:
    """Device-resident cluster snapshot + placement entry points."""

    def __init__(self, device: int = 0, rank: int = 0, world: int = 1, emit_matrix: bool = True,
                 chunk_nodes: int = 0, level_placement: bool = False, committed_levels: bool = False,
                 lw_committed_levels: bool = False, lw_shards: bool = False):
        """level_placement: place exclusive groups at levels >= 1 of set_exclusive_levels (RBGTOPO_CFG_LEVEL_PLACEMENT,
        DESIGN.md §3.9); without it such a group raises RBGTOPO_ELIMIT.  `places_levels` tells callers which it is.
        committed_levels: place_groups_committed places them too, with claims across levels (RBGTOPO_CFG_COMMIT_LEVELS,
        §3.8; implies level_placement).  `places_committed_levels` tells callers which it is.
        lw_committed_levels: place_groups_lw_committed[_ranked] place them too, with claims across levels counted in
        pods (RBGTOPO_CFG_LW_COMMIT_LEVELS, §3.16; implies committed_levels).  `places_lw_committed_levels` tells
        callers which it is.
        lw_shards: place_groups_lw[_committed] also place at world > 1, every rank returning the world = 1 results
        (RBGTOPO_CFG_LW_SHARDS, §3.18); without it they raise RBGTOPO_ELIMIT there.  `places_lw_sharded` tells
        callers which it is."""
        self.lib = _lib.load()
        committed_levels = committed_levels or lw_committed_levels
        level_placement = level_placement or committed_levels
        flags = ((_lib.CFG_LEVEL_PLACEMENT if level_placement else 0) | (_lib.CFG_COMMIT_LEVELS if committed_levels else 0)
                 | (_lib.CFG_LW_COMMIT_LEVELS if lw_committed_levels else 0) | (_lib.CFG_LW_SHARDS if lw_shards else 0))
        cfg = _lib.Config(device=device, rank=rank, world=world, slots=0,
                          emit_matrix=1 if emit_matrix else 0, chunk_nodes=chunk_nodes, flags=flags)
        self.places_levels = bool(level_placement)
        self.places_committed_levels = bool(committed_levels)
        self.places_lw_committed_levels = bool(lw_committed_levels)
        self.places_lw_sharded = bool(lw_shards)
        self.places_lw_ranked = True   # place_groups_lw_ranked: alternates for leader-worker pods (DESIGN.md §3.12)
        self.places_lw_committed = True  # place_groups_lw_committed: committed leader-worker batches (§3.13)
        self.places_committed_ranked = True  # place_groups_committed_ranked: alternates of committed batches (§3.14)
        self.places_lw_committed_ranked = True  # place_groups_lw_committed_ranked: alternates of committed LW batches (§3.15)
        # place_groups[_committed]_ranked_sharded: ranked alternates on node-axis shards, any world (§3.17)
        self.places_sharded_ranked = True
        # set_node_classes + place_groups_eligible[_ranked]: node eligibility per role (§3.19), world = 1 only
        self.places_eligible = world == 1
        # place_groups_eligible_committed[_ranked]: node eligibility in committed batches (§3.20), world = 1 only
        self.places_eligible_committed = world == 1
        h = C.c_void_p()
        self._h = None
        # blob totals of every live staged handle (fetch sizes its outputs from them); created here, not on the first
        # stage, so that threads staging on a new placer all write into the same dict
        self._staged_totals = {}
        self._check(self.lib.rbgtopo_create(C.byref(cfg), C.byref(h)))
        self._h = h
        self.n_nodes = 0
        self.world = world

    # -- plumbing
    def _check(self, rc: int) -> None:
        if rc != 0:
            buf = C.create_string_buffer(512)
            self.lib.rbgtopo_last_error(self._h, buf, 512)
            raise RbgTopoError(rc, buf.value.decode(errors="replace"))

    def close(self) -> None:
        if self._h is not None:
            self.lib.rbgtopo_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- snapshot
    def set_topology(self, row_ptr, col_idx, edge_w, free, domain, domain_owner, generation: int = 0) -> None:
        row_ptr, col_idx, edge_w = _i32(row_ptr), _i32(col_idx), _i32(edge_w)
        free, domain, owner = _i32(free), _i32(domain), _i32(domain_owner)
        n = len(row_ptr) - 1
        self._check(self.lib.rbgtopo_set_topology(self._h, n, len(col_idx), _p(row_ptr), _p(col_idx), _p(edge_w),
                                                  _p(free), _p(domain), len(owner), _p(owner), generation))
        self.n_nodes = n
        self._n_levels = 0   # a new topology leaves occupancy mode

    def update_nodes(self, free=None, domain_owner=None, generation: int = 0) -> None:
        f = None if free is None else _i32(free)
        o = None if domain_owner is None else _i32(domain_owner)
        self._check(self.lib.rbgtopo_update_nodes(self._h, _p(f), _p(o), generation))

    def update_nodes_delta(self, nodes, free, generation: int = 0) -> None:
        """Capacity of a few nodes changed: incremental refresh of base and of the background order."""
        nd, fr = _i32(nodes), _i32(free)
        assert len(nd) == len(fr)
        self._check(self.lib.rbgtopo_update_nodes_delta(self._h, len(nd), _p(nd), _p(fr), generation))

    def set_exclusive_levels(self, level_domain, occupancy, generation: int = 0, level_n_domains=None) -> None:
        """Occupancy mode (DESIGN.md §3.9).  level_domain: [n_levels][n_nodes] domains of levels 1..n_levels (a list
        of per-level vectors or a 2-D array; an empty list = level 0 only), or None to keep the installed partitions
        and refresh the occupancy only.  occupancy: (node, gid, level) per pod carrying the exclusive label.
        level_n_domains: domains per level (default: largest domain id + 1)."""
        occ = _i32(np.asarray(occupancy, dtype=np.int64).reshape(-1, 3))
        if level_domain is None:
            n_levels = getattr(self, "_n_levels", 0)
            lv = nd = None
        else:
            lv = _i32(np.asarray(level_domain, dtype=np.int64).reshape(-1, self.n_nodes))
            n_levels = lv.shape[0]
            nd = _i32(level_n_domains if level_n_domains is not None else [int(r.max()) + 1 for r in lv])
            if not n_levels:   # install "no levels above 0": a non-NULL level_domain with n_levels = 0
                lv, nd = np.zeros(1, dtype=np.int32), None
        self._check(self.lib.rbgtopo_set_exclusive_levels(self._h, n_levels, _p(lv), _p(nd), len(occ), _p(occ),
                                                          generation))
        self._n_levels = n_levels

    def set_node_classes(self, node_class, n_classes: int = None, generation: int = 0) -> None:
        """Node classes (DESIGN.md §3.19): node_class[n] in [0, n_classes) for every node (n_classes defaults to the
        largest class + 1).  Read only by place_groups_eligible[_ranked]; set_topology drops them."""
        cls = _i32(node_class)
        if self.n_nodes and len(cls) != self.n_nodes:   # no topology yet: the library answers RBGTOPO_ENOTOPO
            raise ValueError(f"node_class has {len(cls)} entries for {self.n_nodes} nodes")
        k = int(n_classes) if n_classes is not None else (int(cls.max()) + 1 if len(cls) else 0)
        self._check(self.lib.rbgtopo_set_node_classes(self._h, k, _p(cls), generation))

    # -- hot path, host buffers in/out
    def score_assign(self, blob: np.ndarray) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        blob = _i32(blob)
        ns, tr, _ = blob_totals(blob)
        assign = np.empty(max(tr, 1), dtype=np.int32)
        status = np.empty(max(ns, 1), dtype=np.int32)
        domain = np.empty(max(ns, 1), dtype=np.int32)
        self._check(self.lib.rbgtopo_score_assign(self._h, _p(blob), len(blob), _p(assign), _p(status), _p(domain)))
        return assign[:tr], status[:ns], domain[:ns]

    def place_groups(self, groups_blob: np.ndarray) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """Whole groups, all dependency levels (C++ wave loop behind the ABI)."""
        gb = _i32(groups_blob)
        ng, tp = int(gb[2]), int(gb[4])
        assign = np.empty(max(tp, 1), dtype=np.int32)
        status = np.empty(max(ng, 1), dtype=np.int32)
        domain = np.empty(max(ng, 1), dtype=np.int32)
        self._check(self.lib.rbgtopo_place_groups(self._h, _p(gb), len(gb), _p(assign), _p(status), _p(domain)))
        return assign[:tp], status[:ng], domain[:ng]

    def place_groups_committed(self, groups_blob: np.ndarray) -> Tuple[np.ndarray, np.ndarray, np.ndarray, int]:
        """Whole groups as a committed batch (DESIGN.md §3.8): in blob order, each group sees the capacity and the
        exclusive domains the groups before it took.  Returns (assign, status, domain, selection rounds run)."""
        gb = _i32(groups_blob)
        ng, tp = int(gb[2]), int(gb[4])
        assign = np.empty(max(tp, 1), dtype=np.int32)
        status = np.empty(max(ng, 1), dtype=np.int32)
        domain = np.empty(max(ng, 1), dtype=np.int32)
        rounds = C.c_int32()
        self._check(self.lib.rbgtopo_place_groups_committed(self._h, _p(gb), len(gb), _p(assign), _p(status),
                                                            _p(domain), C.byref(rounds)))
        return assign[:tp], status[:ng], domain[:ng], rounds.value

    def place_groups_committed_ranked(self, groups_blob: np.ndarray, n_alt: int):
        """place_groups_committed plus ranked alternates (DESIGN.md §3.14): returns (assign, status, domain, rounds,
        score[R], alt_node[R, n_alt], alt_score[R, n_alt]).  assign / status / domain / rounds are those of
        place_groups_committed; alt_node[r] holds the next-best nodes of replica r's row that still have room once the
        WHOLE batch is placed and, for a participating role, that no exclusive claim of another gid in the batch
        forbids (-1 / -inf where there are fewer), nothing for unplaced and gang-failed replicas."""
        gb = _i32(groups_blob)
        ng, tp = int(gb[2]), int(gb[4])
        assign = np.empty(max(tp, 1), dtype=np.int32)
        status = np.empty(max(ng, 1), dtype=np.int32)
        domain = np.empty(max(ng, 1), dtype=np.int32)
        rounds = C.c_int32()
        score = np.empty(max(tp, 1), dtype=np.float32)
        alt_node = np.empty((max(tp, 1), max(n_alt, 0)), dtype=np.int32)
        alt_score = np.empty((max(tp, 1), max(n_alt, 0)), dtype=np.float32)
        self._check(self.lib.rbgtopo_place_groups_committed_ranked(
            self._h, _p(gb), len(gb), int(n_alt), _p(assign), _p(status), _p(domain), C.byref(rounds),
            _p(score, _lib.f32p), _p(alt_node) if n_alt > 0 else None, _p(alt_score, _lib.f32p) if n_alt > 0 else None))
        return (assign[:tp], status[:ng], domain[:ng], rounds.value, score[:tp], alt_node[:tp], alt_score[:tp])

    def place_groups_ranked(self, groups_blob: np.ndarray, n_alt: int):
        """place_groups plus ranked alternates (DESIGN.md §3.10): returns (assign, status, domain, score[R],
        alt_node[R, n_alt], alt_score[R, n_alt]).  assign / status / domain are those of place_groups; score[r] is
        replica r's dense-row score at its node, alt_node[r] the next-best nodes of its row that still have room once
        its group is placed (-1 / -inf where there are fewer), nothing for unplaced and gang-failed replicas."""
        gb = _i32(groups_blob)
        ng, tp = int(gb[2]), int(gb[4])
        assign = np.empty(max(tp, 1), dtype=np.int32)
        status = np.empty(max(ng, 1), dtype=np.int32)
        domain = np.empty(max(ng, 1), dtype=np.int32)
        score = np.empty(max(tp, 1), dtype=np.float32)
        alt_node = np.empty((max(tp, 1), max(n_alt, 0)), dtype=np.int32)
        alt_score = np.empty((max(tp, 1), max(n_alt, 0)), dtype=np.float32)
        self._check(self.lib.rbgtopo_place_groups_ranked(
            self._h, _p(gb), len(gb), int(n_alt), _p(assign), _p(status), _p(domain), _p(score, _lib.f32p),
            _p(alt_node) if n_alt > 0 else None, _p(alt_score, _lib.f32p) if n_alt > 0 else None))
        return assign[:tp], status[:ng], domain[:ng], score[:tp], alt_node[:tp], alt_score[:tp]

    @staticmethod
    def _lw_pods(gb: np.ndarray, rp: np.ndarray) -> int:
        """Pods of the assign vector (sum of pending * S); read defensively, the library validates."""
        ng, pods = int(gb[2]), 0
        if len(rp) % 2 == 0 and len(gb) >= 8:
            S = rp[0::2].astype(np.int64)
            k = 0
            for g in range(ng):
                rec = 8 + 12 * g
                if rec + 12 > len(gb):
                    break
                q, role_off = int(gb[rec + 3]), int(gb[rec + 4])
                if q < 0 or k + q > len(S) or role_off < 0 or role_off + 4 * q > len(gb):
                    break
                pods += int((gb[role_off + 1:role_off + 4 * q:4].astype(np.int64) * np.maximum(S[k:k + q], 0)).sum())
                k += q
        return pods

    def place_groups_lw(self, groups_blob: np.ndarray, role_pods) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """Leader-worker replicas (DESIGN.md §3.11): role_pods holds (S, C) per role of every group in blob order —
        S pods per replica, all inside one domain of co-location level C (-1: none).  Returns (assign per pod in
        (group, role, ordinal, pod) order, status, domain)."""
        gb = _i32(groups_blob)
        rp = _i32(np.asarray(role_pods, dtype=np.int64).reshape(-1))
        ng, pods = int(gb[2]), self._lw_pods(gb, rp)
        assign = np.empty(max(pods, 1), dtype=np.int32)
        status = np.empty(max(ng, 1), dtype=np.int32)
        domain = np.empty(max(ng, 1), dtype=np.int32)
        self._check(self.lib.rbgtopo_place_groups_lw(self._h, _p(gb), len(gb), _p(rp), len(rp), _p(assign),
                                                     _p(status), _p(domain)))
        return assign[:pods], status[:ng], domain[:ng]

    def place_groups_lw_committed(self, groups_blob: np.ndarray, role_pods):
        """place_groups_lw as a committed batch (DESIGN.md §3.13): in blob order, each group sees the pods and the
        exclusive domains the groups before it took.  Returns (assign per pod, status, domain, wave-loop rounds run)."""
        gb = _i32(groups_blob)
        rp = _i32(np.asarray(role_pods, dtype=np.int64).reshape(-1))
        ng, pods = int(gb[2]), self._lw_pods(gb, rp)
        assign = np.empty(max(pods, 1), dtype=np.int32)
        status = np.empty(max(ng, 1), dtype=np.int32)
        domain = np.empty(max(ng, 1), dtype=np.int32)
        rounds = C.c_int32()
        self._check(self.lib.rbgtopo_place_groups_lw_committed(self._h, _p(gb), len(gb), _p(rp), len(rp), _p(assign),
                                                               _p(status), _p(domain), C.byref(rounds)))
        return assign[:pods], status[:ng], domain[:ng], rounds.value

    def place_groups_lw_committed_ranked(self, groups_blob: np.ndarray, role_pods, n_alt: int):
        """place_groups_lw_committed plus ranked alternates per pod (DESIGN.md §3.15): returns (assign, status, domain,
        rounds, score[P], alt_node[P, n_alt], alt_score[P, n_alt]).  assign / status / domain / rounds are those of
        place_groups_lw_committed; alt_node[p] holds the next-best nodes of pod p's row that still have room once the
        WHOLE batch is placed, that no exclusive claim of another gid in the batch forbids for a participating role,
        and that keep the replica in its co-location domain (-1 / -inf where there are fewer), nothing for unplaced
        pods and gang-failed groups."""
        gb = _i32(groups_blob)
        rp = _i32(np.asarray(role_pods, dtype=np.int64).reshape(-1))
        ng, pods = int(gb[2]), self._lw_pods(gb, rp)
        assign = np.empty(max(pods, 1), dtype=np.int32)
        status = np.empty(max(ng, 1), dtype=np.int32)
        domain = np.empty(max(ng, 1), dtype=np.int32)
        rounds = C.c_int32()
        score = np.empty(max(pods, 1), dtype=np.float32)
        alt_node = np.empty((max(pods, 1), max(n_alt, 0)), dtype=np.int32)
        alt_score = np.empty((max(pods, 1), max(n_alt, 0)), dtype=np.float32)
        self._check(self.lib.rbgtopo_place_groups_lw_committed_ranked(
            self._h, _p(gb), len(gb), _p(rp), len(rp), int(n_alt), _p(assign), _p(status), _p(domain), C.byref(rounds),
            _p(score, _lib.f32p), _p(alt_node) if n_alt > 0 else None, _p(alt_score, _lib.f32p) if n_alt > 0 else None))
        return (assign[:pods], status[:ng], domain[:ng], rounds.value, score[:pods], alt_node[:pods],
                alt_score[:pods])

    def place_groups_lw_ranked(self, groups_blob: np.ndarray, role_pods, n_alt: int):
        """place_groups_lw plus ranked alternates per pod (DESIGN.md §3.12): returns (assign, status, domain,
        score[P], alt_node[P, n_alt], alt_score[P, n_alt]).  assign / status / domain are those of place_groups_lw;
        score[p] is pod p's dense-row score at its node, alt_node[p] the next-best nodes of its row that still have
        room once its group is placed and that keep the replica in its co-location domain (-1 / -inf where there are
        fewer), nothing for unplaced pods and gang-failed groups."""
        gb = _i32(groups_blob)
        rp = _i32(np.asarray(role_pods, dtype=np.int64).reshape(-1))
        ng, pods = int(gb[2]), self._lw_pods(gb, rp)
        assign = np.empty(max(pods, 1), dtype=np.int32)
        status = np.empty(max(ng, 1), dtype=np.int32)
        domain = np.empty(max(ng, 1), dtype=np.int32)
        score = np.empty(max(pods, 1), dtype=np.float32)
        alt_node = np.empty((max(pods, 1), max(n_alt, 0)), dtype=np.int32)
        alt_score = np.empty((max(pods, 1), max(n_alt, 0)), dtype=np.float32)
        self._check(self.lib.rbgtopo_place_groups_lw_ranked(
            self._h, _p(gb), len(gb), _p(rp), len(rp), int(n_alt), _p(assign), _p(status), _p(domain),
            _p(score, _lib.f32p), _p(alt_node) if n_alt > 0 else None, _p(alt_score, _lib.f32p) if n_alt > 0 else None))
        return assign[:pods], status[:ng], domain[:ng], score[:pods], alt_node[:pods], alt_score[:pods]

    def _eligible_args(self, groups_blob, role_pods, role_admit):
        gb = _i32(groups_blob)
        rp = None if role_pods is None else _i32(np.asarray(role_pods, dtype=np.int64).reshape(-1))
        admit = np.ascontiguousarray(np.asarray(role_admit, dtype=np.uint64).reshape(-1))
        pods = int(gb[4]) if rp is None else self._lw_pods(gb, rp)
        return gb, rp, admit, int(gb[2]), pods

    def place_groups_eligible(self, groups_blob: np.ndarray, role_pods, role_admit):
        """place_groups_lw with node eligibility (DESIGN.md §3.19): role_admit holds one uint64 class mask per role of
        every group in blob order; a role places pods only on nodes whose class bit is set.  role_pods None: one pod
        per replica, no co-location (assign in place_groups order).  Returns (assign, status, domain)."""
        gb, rp, admit, ng, pods = self._eligible_args(groups_blob, role_pods, role_admit)
        assign = np.empty(max(pods, 1), dtype=np.int32)
        status = np.empty(max(ng, 1), dtype=np.int32)
        domain = np.empty(max(ng, 1), dtype=np.int32)
        self._check(self.lib.rbgtopo_place_groups_eligible(
            self._h, _p(gb), len(gb), _p(rp), 0 if rp is None else len(rp), _p(admit, _lib.u64p), len(admit),
            _p(assign), _p(status), _p(domain)))
        return assign[:pods], status[:ng], domain[:ng]

    def place_groups_eligible_ranked(self, groups_blob: np.ndarray, role_pods, role_admit, n_alt: int):
        """place_groups_eligible plus ranked alternates per pod (§3.19, as place_groups_lw_ranked): returns (assign,
        status, domain, score, alt_node, alt_score); no alternate lies on a node the pod's role does not admit."""
        gb, rp, admit, ng, pods = self._eligible_args(groups_blob, role_pods, role_admit)
        assign = np.empty(max(pods, 1), dtype=np.int32)
        status = np.empty(max(ng, 1), dtype=np.int32)
        domain = np.empty(max(ng, 1), dtype=np.int32)
        score = np.empty(max(pods, 1), dtype=np.float32)
        alt_node = np.empty((max(pods, 1), max(n_alt, 0)), dtype=np.int32)
        alt_score = np.empty((max(pods, 1), max(n_alt, 0)), dtype=np.float32)
        self._check(self.lib.rbgtopo_place_groups_eligible_ranked(
            self._h, _p(gb), len(gb), _p(rp), 0 if rp is None else len(rp), _p(admit, _lib.u64p), len(admit),
            int(n_alt), _p(assign), _p(status), _p(domain), _p(score, _lib.f32p),
            _p(alt_node) if n_alt > 0 else None, _p(alt_score, _lib.f32p) if n_alt > 0 else None))
        return assign[:pods], status[:ng], domain[:ng], score[:pods], alt_node[:pods], alt_score[:pods]

    def place_groups_eligible_committed(self, groups_blob: np.ndarray, role_pods, role_admit):
        """place_groups_eligible as a committed batch (DESIGN.md §3.20): in blob order, each group sees the pods and
        the exclusive domains the groups before it took, and every role stays on the nodes its mask admits.  Returns
        (assign, status, domain, wave-loop rounds run)."""
        gb, rp, admit, ng, pods = self._eligible_args(groups_blob, role_pods, role_admit)
        assign = np.empty(max(pods, 1), dtype=np.int32)
        status = np.empty(max(ng, 1), dtype=np.int32)
        domain = np.empty(max(ng, 1), dtype=np.int32)
        rounds = C.c_int32()
        self._check(self.lib.rbgtopo_place_groups_eligible_committed(
            self._h, _p(gb), len(gb), _p(rp), 0 if rp is None else len(rp), _p(admit, _lib.u64p), len(admit),
            _p(assign), _p(status), _p(domain), C.byref(rounds)))
        return assign[:pods], status[:ng], domain[:ng], rounds.value

    def place_groups_eligible_committed_ranked(self, groups_blob: np.ndarray, role_pods, role_admit, n_alt: int):
        """place_groups_eligible_committed plus ranked alternates per pod (§3.20, as place_groups_lw_committed_ranked):
        returns (assign, status, domain, rounds, score, alt_node, alt_score); no alternate lies on a node the pod's
        role does not admit."""
        gb, rp, admit, ng, pods = self._eligible_args(groups_blob, role_pods, role_admit)
        assign = np.empty(max(pods, 1), dtype=np.int32)
        status = np.empty(max(ng, 1), dtype=np.int32)
        domain = np.empty(max(ng, 1), dtype=np.int32)
        rounds = C.c_int32()
        score = np.empty(max(pods, 1), dtype=np.float32)
        alt_node = np.empty((max(pods, 1), max(n_alt, 0)), dtype=np.int32)
        alt_score = np.empty((max(pods, 1), max(n_alt, 0)), dtype=np.float32)
        self._check(self.lib.rbgtopo_place_groups_eligible_committed_ranked(
            self._h, _p(gb), len(gb), _p(rp), 0 if rp is None else len(rp), _p(admit, _lib.u64p), len(admit),
            int(n_alt), _p(assign), _p(status), _p(domain), C.byref(rounds), _p(score, _lib.f32p),
            _p(alt_node) if n_alt > 0 else None, _p(alt_score, _lib.f32p) if n_alt > 0 else None))
        return (assign[:pods], status[:ng], domain[:ng], rounds.value, score[:pods], alt_node[:pods],
                alt_score[:pods])

    # -- staged (device-resident) batches
    def stage(self, blob: np.ndarray) -> int:
        blob = _i32(blob)
        h = C.c_int32(-1)
        self._check(self.lib.rbgtopo_stage(self._h, _p(blob), len(blob), C.byref(h)))
        self._staged_totals[h.value] = blob_totals(blob)
        return h.value

    def stage_groups(self, groups_blob: np.ndarray) -> int:
        """Compile whole groups into a device-resident multi-wave plan (see rbgtopo.h)."""
        gb = _i32(groups_blob)
        h = C.c_int32(-1)
        self._check(self.lib.rbgtopo_stage_groups(self._h, _p(gb), len(gb), C.byref(h)))
        self._staged_totals[h.value] = (int(gb[2]), int(gb[4]), 0)   # fetch: per group / per pending replica
        return h.value

    def run_staged(self, handle: int, iters: int = 1) -> None:
        self._check(self.lib.rbgtopo_run_staged(self._h, handle, iters))

    def run_staged_chain(self, handles, passes: int) -> None:
        """`passes` passes round robin over distinct staged GROUPS batches, enqueue only: the dense-matrix kernel of
        a pass is chained behind the selection kernel of the pass before it (rbgtopo_run_staged_chain)."""
        hs = np.ascontiguousarray(handles, dtype=np.int32)
        self._check(self.lib.rbgtopo_run_staged_chain(self._h, _p(hs), len(hs), passes))

    def fetch(self, handle: int):
        ns, tr, _ = self._staged_totals[handle]
        assign = np.empty(max(tr, 1), dtype=np.int32)
        status = np.empty(max(ns, 1), dtype=np.int32)
        domain = np.empty(max(ns, 1), dtype=np.int32)
        self._check(self.lib.rbgtopo_fetch(self._h, handle, _p(assign), _p(status), _p(domain)))
        return assign[:tr], status[:ns], domain[:ns]

    def release(self, handle: int) -> None:
        # Handle ids are pool slots: once rbgtopo_release returns, another thread's stage can receive the same id and
        # store its totals.  Dropping ours first keeps that thread's entry; a refused release puts ours back.
        totals = self._staged_totals.pop(handle, None)
        rc = self.lib.rbgtopo_release(self._h, handle)
        if rc != 0 and totals is not None:
            self._staged_totals[handle] = totals
        self._check(rc)

    def read_scores(self, handle: int, row: int) -> np.ndarray:
        lo, hi = self.slab()
        out = np.empty(hi - lo, dtype=np.float32)
        self._check(self.lib.rbgtopo_read_scores(self._h, handle, row, _p(out, _lib.f32p), len(out)))
        return out

    def read_topk(self, handle: int, rolerow: int, k: int = 32) -> np.ndarray:
        out = np.zeros(k, dtype=np.uint64)
        self._check(self.lib.rbgtopo_read_topk(self._h, handle, rolerow, _p(out, _lib.u64p), k))
        return out

    SNAPSHOT = {"base": (0, np.float32), "order": (1, np.uint64), "order_all": (2, np.uint64), "pos": (3, np.int32),
                "delta_repairs": (4, np.int64), "level_owner": (5, np.int32)}

    def read_snapshot(self, what: str) -> np.ndarray:
        """One per-snapshot vector exactly as the device holds it (rbgtopo_read_snapshot): "base", "order" (this
        rank's slab), "order_all", "pos" (world == 1), "delta_repairs" (one int64) or "level_owner" (occupancy mode:
        [n_levels + 1][n_nodes], empty outside it)."""
        code, dt = self.SNAPSHOT[what]
        n = C.c_int64()
        rc = self.lib.rbgtopo_read_snapshot(self._h, code, None, 0, C.byref(n))   # sizes only: EINVAL unless empty
        if rc not in (0, -1):
            self._check(rc)
        out = np.empty(n.value, dtype=dt)
        self._check(self.lib.rbgtopo_read_snapshot(self._h, code, out.ctypes.data_as(C.c_void_p), out.nbytes, C.byref(n)))
        return out.reshape(-1, self.n_nodes) if what == "level_owner" else out

    # -- node-axis sharding
    def slab(self) -> Tuple[int, int]:
        lo, hi = C.c_int32(), C.c_int32()
        self._check(self.lib.rbgtopo_slab(self._h, C.byref(lo), C.byref(hi)))
        return lo.value, hi.value

    def shard_waves(self, handle: int) -> int:
        n = C.c_int32()
        self._check(self.lib.rbgtopo_shard_waves(self._h, handle, C.byref(n)))
        return n.value

    def shard_wave_score(self, handle: int, wave: int) -> Tuple[int, int]:
        p, nb = C.c_void_p(), C.c_int64()
        self._check(self.lib.rbgtopo_shard_wave_score(self._h, handle, wave, C.byref(p), C.byref(nb)))
        return p.value, nb.value

    def shard_wave_merge(self, handle: int, wave: int, keys_all_ptr: int) -> Tuple[bool, int, int]:
        need, p, nb = C.c_int32(), C.c_void_p(), C.c_int64()
        self._check(self.lib.rbgtopo_shard_wave_merge(self._h, handle, wave, C.c_void_p(keys_all_ptr), C.byref(need),
                                                      C.byref(p), C.byref(nb)))
        return bool(need.value), p.value, nb.value

    def shard_wave_assign(self, handle: int, wave: int, keys2_all_ptr: Optional[int]) -> None:
        self._check(self.lib.rbgtopo_shard_wave_assign(self._h, handle, wave,
                                                       C.c_void_p(keys2_all_ptr) if keys2_all_ptr else None))

    def shard_score(self, handle: int) -> Tuple[int, int]:
        p, nb = C.c_void_p(), C.c_int64()
        self._check(self.lib.rbgtopo_shard_score(self._h, handle, C.byref(p), C.byref(nb)))
        return p.value, nb.value

    def shard_merge(self, handle: int, keys_all_ptr: int) -> Tuple[bool, int, int]:
        need, p, nb = C.c_int32(), C.c_void_p(), C.c_int64()
        self._check(self.lib.rbgtopo_shard_merge(self._h, handle, C.c_void_p(keys_all_ptr), C.byref(need),
                                                 C.byref(p), C.byref(nb)))
        return bool(need.value), p.value, nb.value

    def shard_assign(self, handle: int, keys2_all_ptr: Optional[int]) -> None:
        self._check(self.lib.rbgtopo_shard_assign(self._h, handle,
                                                  C.c_void_p(keys2_all_ptr) if keys2_all_ptr else None))

    # -- ranked alternates on node-axis shards (DESIGN.md §3.17)
    def shard_place_groups_ranked(self, groups_blob: np.ndarray, n_alt: int):
        """Local half of place_groups_ranked on this rank: (assign, status, domain, xhandle, keys_ptr, keys_bytes).
        keys_ptr / keys_bytes: this rank's exchange buffer (library-owned device memory) for the all-gather."""
        gb = _i32(groups_blob)
        ng, tp = int(gb[2]), int(gb[4])
        assign = np.empty(max(tp, 1), dtype=np.int32)
        status = np.empty(max(ng, 1), dtype=np.int32)
        domain = np.empty(max(ng, 1), dtype=np.int32)
        xh, p, nb = C.c_int32(), C.c_void_p(), C.c_int64()
        self._check(self.lib.rbgtopo_shard_place_groups_ranked(
            self._h, _p(gb), len(gb), int(n_alt), _p(assign), _p(status), _p(domain), C.byref(xh), C.byref(p),
            C.byref(nb)))
        return assign[:tp], status[:ng], domain[:ng], xh.value, p.value, nb.value

    def shard_place_groups_committed_ranked(self, groups_blob: np.ndarray, n_alt: int):
        """Local half of place_groups_committed_ranked: (assign, status, domain, rounds, xhandle, keys_ptr,
        keys_bytes)."""
        gb = _i32(groups_blob)
        ng, tp = int(gb[2]), int(gb[4])
        assign = np.empty(max(tp, 1), dtype=np.int32)
        status = np.empty(max(ng, 1), dtype=np.int32)
        domain = np.empty(max(ng, 1), dtype=np.int32)
        rounds, xh, p, nb = C.c_int32(), C.c_int32(), C.c_void_p(), C.c_int64()
        self._check(self.lib.rbgtopo_shard_place_groups_committed_ranked(
            self._h, _p(gb), len(gb), int(n_alt), _p(assign), _p(status), _p(domain), C.byref(rounds), C.byref(xh),
            C.byref(p), C.byref(nb)))
        return assign[:tp], status[:ng], domain[:ng], rounds.value, xh.value, p.value, nb.value

    def shard_place_groups_lw_ranked(self, groups_blob: np.ndarray, role_pods, n_alt: int):
        """Local half of place_groups_lw_ranked (DESIGN.md §3.18): (assign per pod, status, domain, xhandle, keys_ptr,
        keys_bytes)."""
        gb = _i32(groups_blob)
        rp = _i32(np.asarray(role_pods, dtype=np.int64).reshape(-1))
        ng, pods = int(gb[2]), self._lw_pods(gb, rp)
        assign = np.empty(max(pods, 1), dtype=np.int32)
        status = np.empty(max(ng, 1), dtype=np.int32)
        domain = np.empty(max(ng, 1), dtype=np.int32)
        xh, p, nb = C.c_int32(), C.c_void_p(), C.c_int64()
        self._check(self.lib.rbgtopo_shard_place_groups_lw_ranked(
            self._h, _p(gb), len(gb), _p(rp), len(rp), int(n_alt), _p(assign), _p(status), _p(domain), C.byref(xh),
            C.byref(p), C.byref(nb)))
        return assign[:pods], status[:ng], domain[:ng], xh.value, p.value, nb.value

    def shard_place_groups_lw_committed_ranked(self, groups_blob: np.ndarray, role_pods, n_alt: int):
        """Local half of place_groups_lw_committed_ranked (§3.18): (assign per pod, status, domain, rounds, xhandle,
        keys_ptr, keys_bytes)."""
        gb = _i32(groups_blob)
        rp = _i32(np.asarray(role_pods, dtype=np.int64).reshape(-1))
        ng, pods = int(gb[2]), self._lw_pods(gb, rp)
        assign = np.empty(max(pods, 1), dtype=np.int32)
        status = np.empty(max(ng, 1), dtype=np.int32)
        domain = np.empty(max(ng, 1), dtype=np.int32)
        rounds, xh, p, nb = C.c_int32(), C.c_int32(), C.c_void_p(), C.c_int64()
        self._check(self.lib.rbgtopo_shard_place_groups_lw_committed_ranked(
            self._h, _p(gb), len(gb), _p(rp), len(rp), int(n_alt), _p(assign), _p(status), _p(domain),
            C.byref(rounds), C.byref(xh), C.byref(p), C.byref(nb)))
        return assign[:pods], status[:ng], domain[:ng], rounds.value, xh.value, p.value, nb.value

    def shard_alternates_merge(self, xhandle: int, keys_all_ptr: int, n_replicas: int, n_alt: int):
        """Merge half: (score[R], alt_node[R, n_alt], alt_score[R, n_alt]) from the gathered buffers (world x
        keys_bytes, rank-major, device memory).  Consumes the handle."""
        R = int(n_replicas)
        score = np.empty(max(R, 1), dtype=np.float32)
        alt_node = np.empty((max(R, 1), max(n_alt, 0)), dtype=np.int32)
        alt_score = np.empty((max(R, 1), max(n_alt, 0)), dtype=np.float32)
        self._check(self.lib.rbgtopo_shard_alternates_merge(
            self._h, int(xhandle), C.c_void_p(keys_all_ptr), _p(score, _lib.f32p), _p(alt_node) if n_alt > 0 else None,
            _p(alt_score, _lib.f32p) if n_alt > 0 else None))
        return score[:R], alt_node[:R], alt_score[:R]

    def _default_all_gather(self, ptr: int, nbytes: int):
        """torch.distributed.all_gather_into_tensor of this rank's exchange buffer over the default process group."""
        import torch
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized()):
            raise RuntimeError("a sharded ranked placement at world > 1 needs all_gather= or an initialised "
                               "torch.distributed process group")
        dev = torch.device("cuda", torch.cuda.current_device())
        mine = torch.as_tensor(_DevBytes(ptr, nbytes), device=dev)
        out = torch.empty(self.world * nbytes, dtype=torch.uint8, device=dev)
        dist.all_gather_into_tensor(out, mine)
        return out

    def _sharded(self, local, n_alt: int, all_gather):
        """Local half, all-gather, merge.  all_gather(ptr, nbytes) returns a device buffer of world x nbytes bytes,
        rank-major (a torch tensor, or anything with data_ptr()), complete when its stream is done: the calling
        thread's current torch stream is synchronised before the merge.  The handle is released when it fails."""
        *placed, xh, ptr, nbytes = local
        if self.world == 1 and all_gather is None:
            gathered = None
        else:
            try:
                gathered = (all_gather or self._default_all_gather)(ptr, nbytes)
                import torch
                torch.cuda.current_stream().synchronize()
            except BaseException:
                self.release(xh)
                raise
        keys_all = ptr if gathered is None else int(gathered.data_ptr())
        merged = self.shard_alternates_merge(xh, keys_all, len(placed[0]), n_alt)
        return (*placed, *merged)

    def place_groups_ranked_sharded(self, groups_blob: np.ndarray, n_alt: int, all_gather=None):
        """place_groups_ranked on node-axis shards (DESIGN.md §3.17), valid for any world: every rank calls it with
        the same blob and gets all six outputs of the world = 1 place_groups_ranked, bit for bit.  all_gather(ptr,
        nbytes) -> a device buffer of world x nbytes, rank-major; default: torch.distributed.all_gather_into_tensor
        on the initialised default process group (world = 1 needs none)."""
        return self._sharded(self.shard_place_groups_ranked(groups_blob, n_alt), n_alt, all_gather)

    def place_groups_committed_ranked_sharded(self, groups_blob: np.ndarray, n_alt: int, all_gather=None):
        """place_groups_committed_ranked on node-axis shards (§3.17): (assign, status, domain, rounds, score,
        alt_node, alt_score) as the world = 1 call gives them; all_gather as for place_groups_ranked_sharded."""
        return self._sharded(self.shard_place_groups_committed_ranked(groups_blob, n_alt), n_alt, all_gather)

    def place_groups_lw_ranked_sharded(self, groups_blob: np.ndarray, role_pods, n_alt: int, all_gather=None):
        """place_groups_lw_ranked on node-axis shards (DESIGN.md §3.18), valid for any world: (assign, status, domain,
        score, alt_node, alt_score) per pod as the world = 1 call gives them; all_gather as for
        place_groups_ranked_sharded."""
        return self._sharded(self.shard_place_groups_lw_ranked(groups_blob, role_pods, n_alt), n_alt, all_gather)

    def place_groups_lw_committed_ranked_sharded(self, groups_blob: np.ndarray, role_pods, n_alt: int,
                                                 all_gather=None):
        """place_groups_lw_committed_ranked on node-axis shards (§3.18): (assign, status, domain, rounds, score,
        alt_node, alt_score) per pod as the world = 1 call gives them; all_gather as for place_groups_ranked_sharded."""
        return self._sharded(self.shard_place_groups_lw_committed_ranked(groups_blob, role_pods, n_alt), n_alt,
                             all_gather)

    # -- all-gather over NVLink peer memory inside the library
    def p2p_export(self, rows_cap: int = 0):
        """(64-byte IPC handle, device pointer) of this rank's exchange buffer."""
        buf = C.create_string_buffer(64)
        ptr = C.c_void_p()
        self._check(self.lib.rbgtopo_p2p_export(self._h, rows_cap, buf, 64, C.byref(ptr)))
        return bytes(buf.raw), ptr.value

    def p2p_import(self, handles=None, ptrs=None) -> None:
        """handles: list of `world` 64-byte IPC handles (one process per GPU), or ptrs: list of `world`
        device pointers (contexts of one process)."""
        if ptrs is not None:
            arr = (C.c_void_p * len(ptrs))(*ptrs)
            self._check(self.lib.rbgtopo_p2p_import(self._h, None, arr))
        else:
            blob = b"".join(handles)
            self._check(self.lib.rbgtopo_p2p_import(self._h, C.c_char_p(blob), None))

    def p2p_connect(self, D) -> None:
        """One process per GPU: exchange the IPC handles over torch.distributed (plumbing) and map the peers."""
        import torch
        h, _ = self.p2p_export()
        mine = torch.frombuffer(bytearray(h), dtype=torch.uint8).cuda()
        allh = torch.empty(D.world * 64, dtype=torch.uint8, device="cuda")
        D.dist.all_gather_into_tensor(allh, mine)
        raw = bytes(allh.cpu().numpy().tobytes())
        self.p2p_import(handles=[raw[64 * g: 64 * (g + 1)] for g in range(D.world)])
        D.barrier()

    def run_staged_p2p(self, handle: int, iters: int = 1) -> None:
        self._check(self.lib.rbgtopo_run_staged_p2p(self._h, handle, iters))

    def p2p_stats(self):
        b, t = C.c_int64(), C.c_int32()
        self._check(self.lib.rbgtopo_p2p_stats(self._h, C.byref(b), C.byref(t)))
        return dict(peer_bytes_last_pass=b.value, timed_out=bool(t.value))

    def set_stream(self, cuda_stream: Optional[int]) -> None:
        """None restores the internal per-call streams.  A torch default stream has
        handle 0 (the legacy NULL stream): it is passed as cudaStreamLegacy (0x1)."""
        if cuda_stream is None:
            self._check(self.lib.rbgtopo_set_stream(self._h, None))
        else:
            self._check(self.lib.rbgtopo_set_stream(self._h, C.c_void_p(cuda_stream if cuda_stream else 1)))

    def set_kernel_timing(self, on: bool) -> None:
        """Per-kernel CUDA events inside a pass (serialises the two plan kernels); off = a pass is timed as a
        whole and the selection kernel is a programmatic dependent of the dense-matrix kernel."""
        self._check(self.lib.rbgtopo_set_kernel_timing(self._h, 1 if on else 0))

    # -- stats
    def last_timing(self) -> dict:
        t = _lib.Timing()
        self._check(self.lib.rbgtopo_last_timing(self._h, C.byref(t)))
        return {k: getattr(t, k) for k, _ in _lib.Timing._fields_}

    def last_pass_times(self, cap: int = 4096):
        """(score_ms[], select_ms[]) of the passes the last fetch harvested."""
        a = np.zeros(cap, dtype=np.float32)
        b = np.zeros(cap, dtype=np.float32)
        n = C.c_int32()
        self._check(self.lib.rbgtopo_last_pass_times(self._h, _p(a, _lib.f32p), _p(b, _lib.f32p), cap, C.byref(n)))
        k = min(n.value, cap)
        return a[:k].copy(), b[:k].copy()

    def stats(self) -> dict:
        g, c, s, k = C.c_uint64(), C.c_int64(), C.c_int64(), C.c_int64()
        self._check(self.lib.rbgtopo_stats(self._h, C.byref(g), C.byref(c), C.byref(s), C.byref(k)))
        n, per_sm, rounds = C.c_int32(), C.c_int32(), C.c_int32()
        self._check(self.lib.rbgtopo_plan_occupancy(self._h, C.byref(n), C.byref(per_sm), C.byref(rounds)))
        return dict(generation=g.value, calls=c.value, scores_total=s.value, kernel_launches=k.value,
                    plan_ctas=n.value, plan_ctas_per_sm=per_sm.value, plan_rounds=rounds.value)
