"""Host-side mirror of the reference plugin surface for this path.

The reference's boundary is the Go interface ``scheduler.PodGroupManager``
(pkg/scheduler/podgroup_manager.go:64-78): ``ReconcilePodGroup(ctx, rbg, ...)``
called from step 6 of Reconcile (rolebasedgroup_controller.go:200-204,422-430)
and ``InjectPodGroupLabels(rbg, podTemplate)`` called while the pod template is
built (pkg/reconciler/pod_reconciler.go:150-153).  ``B200TopoPodGroupManager``
keeps those two method names and meanings; the Go shim in INTEGRATION.md is the
same logic over cgo.  Everything numeric goes through the C ABI
(include/rbgtopo.h) — this file only turns RoleBasedGroup specs into placement
steps (levels -> waves) and turns the results into per-replica hints.

Reference semantics used (never re-derived here, all cited):
  - role levels: dependencyOrder, pkg/dependency/dependency.go:129-205
    (via rbgtopo_dependency_levels)
  - group size / gang MinMember: GetGroupSize, api/workloads/v1alpha2/helper.go:50-65
  - pending replicas per role: coordination target - current
    (rolebasedgroup_controller.go:509-518; scaler.go:70-172 via
    rbgtopo_calculate_target_replicas)
  - replica identity "{rbg}-{role}-{ordinal}": helper.go:68-81,
    stateful_instance_set_utils.go:74-76
  - annotations: api/workloads/constants/annotation.go:25,29,37
"""
from __future__ import annotations

import ctypes as C
import json
import logging
from dataclasses import dataclass, field
from typing import Dict, List, Mapping, Optional, Sequence, Tuple

import numpy as np

from . import _lib
from .blob import (MAX_STEP_REPLICAS, MAX_STEP_ROLES, NEED_CAP, ROLE_EXCLUSIVE, STEP_EXCLUSIVE, STEP_GANG,
                   BlobBuilder, Group, GroupsBuilder, Step)
from .engine import TopoPlacer
from .ingest import NodeClasses, NotDecidable, role_admit

RBG_PREFIX = "rbg.workloads.x-k8s.io/"                       # api/workloads/constants
EXCLUSIVE_TOPOLOGY_KEY = RBG_PREFIX + "group-exclusive-topology"   # annotation.go:25
ROLE_DISABLE_EXCLUSIVE_KEY = RBG_PREFIX + "role-disable-exclusive"  # annotation.go:29,60
GANG_SCHEDULING_KEY = RBG_PREFIX + "group-gang-scheduling"          # annotation.go:37
PLACEMENT_HINT_KEY = RBG_PREFIX + "b200-topo-placement"             # new: RoleID -> node map
PLACEMENT_ALTERNATES_KEY = RBG_PREFIX + "b200-topo-alternates"       # new: RoleID -> ranked fallback nodes
COLOCATE_KEY = RBG_PREFIX + "b200-topo-colocate"                     # new, per role: topology key of one replica's pods
SCHEDULER_PLUGIN_NAME = "b200-topo"                                 # --scheduler-name value
# what the wrapped gang plugins inject into the pod template when gang scheduling is on
KUBE_POD_GROUP_LABEL = "pod-group.scheduling.sigs.k8s.io/name"      # k8s-scheduler-plugin/manager.go:49,91-98
VOLCANO_GROUP_ANNOTATION = "scheduling.k8s.io/group-name"           # volcano/manager.go:85-92


@dataclass
class RoleSpec:
    """The fields of v1alpha2.RoleSpec this path reads (rolebasedgroup_types.go:166-229)."""
    name: str
    replicas: int
    dependencies: Sequence[str] = ()
    demand: int = 1                      # accelerator slots per replica (new input)
    lws_size: int = 0                    # LeaderWorkerPattern.Size, 0 = not LWS
    annotations: Dict[str, str] = field(default_factory=dict)
    # the pod template's node eligibility (DESIGN.md §3.19): spec.nodeSelector, the nodeSelectorTerms of
    # affinity.nodeAffinity.requiredDuringSchedulingIgnoredDuringExecution (empty: none), spec.tolerations
    node_selector: Dict[str, str] = field(default_factory=dict)
    node_affinity: Sequence[Mapping] = ()
    tolerations: Sequence[Mapping[str, str]] = ()


@dataclass
class ScalingRule:
    """A CoordinatedPolicyRule with Strategy.Scaling (coordinatedpolicy_types.go:41-45;
    rolebasedgroup_controller.go:981-994): the roles it paces, MaxSkew and Progression."""
    roles: Sequence[str]
    max_skew: str = "100%"
    progression: str = ""               # "" | "OrderScheduled" | "OrderReady" (scaler.go:141-169)


@dataclass
class RoleStatus:
    """What CalculateScalingForAllCoordination reads per role: status.roleStatuses[] and the
    scheduled-pod count of getScheduledReplicas (rolebasedgroup_controller.go:1008-1024, :1057-1080)."""
    replicas: int = 0
    ready: int = 0
    scheduled: int = 0


PROGRESSION = {"": 0, None: 0, "OrderScheduled": 1, "OrderReady": 2}


@dataclass
class RoleBasedGroup:
    namespace: str
    name: str
    roles: List[RoleSpec]
    annotations: Dict[str, str] = field(default_factory=dict)
    gid: int = 0                                             # dense id of the group in the Node cache
    policy_rules: List[Sequence[str]] = field(default_factory=list)  # CoordinatedPolicy role sets
    # status the controller already has at step 5 of Reconcile:
    targets: Optional[Dict[str, int]] = None     # coordination scaling targets (role -> replicas)
    current: Dict[str, int] = field(default_factory=dict)    # status.roleStatuses[].replicas
    placed: List[Tuple[str, int]] = field(default_factory=list)  # (role, node) of scheduled pods
    exclusive_domain: int = -1                   # domain the group already occupies, if any
    # coordination scaling inputs; when `targets` is None and rules exist the targets are computed
    # here with the reference's own arithmetic (rbgtopo_calculate_target_replicas)
    scaling_rules: List[ScalingRule] = field(default_factory=list)
    status: Dict[str, RoleStatus] = field(default_factory=dict)


RBGTOPO_NO_HINT = -1   # Placement.status of a group the manager gives no hint (B200TopoPodGroupManager.no_hint)
ALL_CLASSES = (1 << 64) - 1   # the class mask of a role that admits every node class (DESIGN.md §3.19)


@dataclass
class Placement:
    status: int                      # 0 all placed, 1 partial, 2 gang failed, RBGTOPO_NO_HINT
    nodes: Dict[str, int]            # "{rbg}-{role}-{ordinal}" -> node (-1 = unplaced)
    domain: int = -1
    scores: int = 0                  # (replica x node) scores computed for this group
    alternates: Dict[str, List[int]] = field(default_factory=dict)  # "{rbg}-{role}-{ordinal}" -> next-best nodes


class HostArith:
    """ctypes access to the reference-pinned host arithmetic exported by the ABI."""

    def __init__(self):
        self.lib = _lib.load()

    def group_size(self, roles: Sequence[RoleSpec]) -> int:
        n = len(roles)
        rep = (C.c_int32 * n)(*[r.replicas for r in roles])
        lws = (C.c_int32 * n)(*[r.lws_size for r in roles])
        return self.lib.rbgtopo_group_size(n, rep, lws)

    def dependency_levels(self, roles: Sequence[RoleSpec]) -> List[List[int]]:
        n = len(roles)
        names = [r.name for r in roles]
        index = {nm: i for i, nm in enumerate(names)}
        off, idx = [0], []
        for r in roles:
            for d in r.dependencies:
                if d not in index:
                    raise ValueError(f"role [{r.name}] with dependency role [{d}] not found in rbg")
                idx.append(index[d])
            off.append(len(idx))
        c_names = (C.c_char_p * n)(*[nm.encode() for nm in names])
        c_off = (C.c_int32 * (n + 1))(*off)
        c_idx = (C.c_int32 * max(len(idx), 1))(*idx)
        level = (C.c_int32 * n)()
        order = (C.c_int32 * n)()
        nl = self.lib.rbgtopo_dependency_levels(n, c_names, c_off, c_idx, level, order)
        if nl < 0:
            raise ValueError("failed to sort roles by dependency order: cycle detected")
        out: List[List[int]] = [[] for _ in range(nl)]
        for i in range(n):
            out[level[order[i]]].append(order[i])
        return out

    def parse_percentage(self, s: str) -> float:
        out = C.c_double()
        if self.lib.rbgtopo_parse_percentage(s.encode(), C.byref(out)) != 0:
            raise ValueError(f"invalid maxSkew {s!r}")
        return out.value

    def scaling_targets(self, rbg: "RoleBasedGroup") -> Optional[Dict[str, int]]:
        """CalculateScalingForAllCoordination (rolebasedgroup_controller.go:968-1054): one
        CalculateTargetReplicas per rule with a scaling strategy; a role paced by several rules
        takes the minimum.  None when the group has no scaling rule."""
        if not rbg.scaling_rules:
            return None
        spec = {r.name: r.replicas for r in rbg.roles}
        result: Dict[str, int] = {}
        for rule in rbg.scaling_rules:
            names = list(rule.roles)
            st = [rbg.status.get(nm, RoleStatus()) for nm in names]
            tgt = self.calculate_target_replicas(self.parse_percentage(rule.max_skew), PROGRESSION[rule.progression],
                                                 [spec.get(nm, 0) for nm in names], [s.replicas for s in st],
                                                 [s.scheduled for s in st], [s.ready for s in st])
            for nm, t in zip(names, tgt):
                result[nm] = min(result[nm], t) if nm in result else t
        return result

    def calculate_target_replicas(self, max_skew: float, progression: int, desired, current, scheduled, ready):
        n = len(desired)
        arr = lambda v: (C.c_int32 * n)(*v)
        tgt = (C.c_int32 * n)()
        rc = self.lib.rbgtopo_calculate_target_replicas(max_skew, progression, n, arr(desired), arr(current),
                                                        arr(scheduled), arr(ready), tgt)
        if rc != 0:
            raise ValueError("no role states provided")
        return list(tgt)


@dataclass
class _Wave:
    roles: List[Tuple[int, int, int]]   # (role index, first ordinal, count)


class _GroupRun:
    """Per-group state while its levels/waves are placed."""

    def __init__(self, rbg: RoleBasedGroup, arith: HostArith, plan_waves: bool = True, excl_level: int = 0):
        self.rbg = rbg
        self.excl_level = excl_level  # index of the group's exclusive key (DESIGN.md §3.9)
        roles = rbg.roles
        self.Q = len(roles)
        index = {r.name: i for i, r in enumerate(roles)}
        # pair matrix (spec §3.2): same role, dependency edge, or shared policy rule
        pair = np.eye(self.Q, dtype=np.int32)
        for i, r in enumerate(roles):
            for d in r.dependencies:
                pair[i, index[d]] = pair[index[d], i] = 1
        for rule in rbg.policy_rules:
            ids = [index[x] for x in rule if x in index]
            for a in ids:
                for b in ids:
                    pair[a, b] = 1
        self.pair = pair
        self.exclusive = EXCLUSIVE_TOPOLOGY_KEY in rbg.annotations
        self.gang = rbg.annotations.get(GANG_SCHEDULING_KEY) == "true"
        self.role_excl = [r.annotations.get(ROLE_DISABLE_EXCLUSIVE_KEY) != "true" for r in roles]
        # pending replicas: coordination target (or spec) minus current
        self.first_ordinal, self.pending = [], []
        targets = rbg.targets if rbg.targets is not None else arith.scaling_targets(rbg)
        for r in roles:
            tgt = r.replicas if targets is None else targets.get(r.name, r.replicas)
            cur = rbg.current.get(r.name, rbg.status[r.name].replicas if r.name in rbg.status else 0)
            self.first_ordinal.append(cur)
            self.pending.append(max(tgt - cur, 0))
        self.unplaced = list(self.pending)
        self.anchors: Dict[Tuple[int, int], int] = {}
        for role_name, node in rbg.placed:
            key = (node, index[role_name])
            self.anchors[key] = self.anchors.get(key, 0) + 1
        self.consumed: Dict[int, int] = {}
        self.fixed_domain = rbg.exclusive_domain
        self.failed = False
        self.result_nodes: Dict[str, int] = {}
        self.status = 0
        self.scores = 0
        # waves: levels in order, roles lexicographic inside a level, packed to the ABI limits
        self.waves: List[_Wave] = []
        levels = arith.dependency_levels(roles)
        self.order = [ri for level in levels for ri in level]        # (level, name) order
        self.level_of = {ri: li for li, level in enumerate(levels) for ri in level}
        for level in (levels if plan_waves else []):
            cur_roles: List[Tuple[int, int, int]] = []
            cur_n = 0
            for ri in level:
                left, ordinal = self.pending[ri], self.first_ordinal[ri]
                while left > 0:
                    room = MAX_STEP_REPLICAS - cur_n
                    if room == 0 or len(cur_roles) == MAX_STEP_ROLES:
                        self.waves.append(_Wave(cur_roles))
                        cur_roles, cur_n = [], 0
                        room = MAX_STEP_REPLICAS
                    take = min(left, room)
                    cur_roles.append((ri, ordinal, take))
                    cur_n += take
                    left -= take
                    ordinal += take
            if cur_roles:
                self.waves.append(_Wave(cur_roles))

    def step(self, w: int) -> Step:
        wave = self.waves[w]
        roles_rec, pair_rows = [], []
        for ri, _, cnt in wave.roles:
            need = 0
            for q in range(self.Q):
                if self.pair[ri, q] > 0:
                    need += self.unplaced[q]
            need = min(NEED_CAP, need)
            flags = ROLE_EXCLUSIVE if self.role_excl[ri] else 0
            roles_rec.append((cnt, self.rbg.roles[ri].demand, need, flags))
            pair_rows.append([int(x) for x in self.pair[ri]])
        flags = (STEP_EXCLUSIVE if self.exclusive else 0) | (STEP_GANG if self.gang else 0)
        return Step(gid=self.rbg.gid, roles=roles_rec, pair=pair_rows,
                    anchors=[(n, q, c) for (n, q), c in sorted(self.anchors.items())],
                    consumed=sorted(self.consumed.items()), flags=flags,
                    fixed_domain=self.fixed_domain if self.exclusive else -1, level=self.excl_level)

    def absorb(self, w: int, assign: np.ndarray, status: int, domain: int, n_nodes: int) -> None:
        wave = self.waves[w]
        k = 0
        self.scores += len(assign) * n_nodes
        for ri, ordinal, cnt in wave.roles:
            role = self.rbg.roles[ri]
            for c in range(cnt):
                node = int(assign[k]); k += 1
                self.result_nodes[f"{self.rbg.name}-{role.name}-{ordinal + c}"] = node
                if node >= 0:
                    self.anchors[(node, ri)] = self.anchors.get((node, ri), 0) + 1
                    self.consumed[node] = self.consumed.get(node, 0) + role.demand
                    self.unplaced[ri] -= 1
        if self.exclusive and domain >= 0 and any(n >= 0 for n in assign):
            self.fixed_domain = domain
        self.status = max(self.status, status)
        if self.gang and status != 0:
            self.failed = True


class B200TopoPodGroupManager:
    """Third ``PodGroupManager`` implementation (plugin type "b200-topo")."""

    def __init__(self, placer: TopoPlacer, inner: Optional[str] = "scheduler-plugins",
                 exclusive_keys: Optional[Sequence[str]] = None, alternates: int = 0, leader_worker: bool = False,
                 all_gather=None, node_classes: Optional[NodeClasses] = None):
        """inner: the gang plugin this manager wraps for the PodGroup CR and the pod-group label —
        "scheduler-plugins" (kube), "volcano" or None (the Go manager takes the implementation object).
        exclusive_keys: the topology keys exclusive groups may name (DESIGN.md §3.9), keys[0] = the level-0 label.
        None: every key is treated as the level-0 label.  With a list, an exclusive group whose key is keys[i] is
        placed at level i (GROUPS word +10, step word +14) when the placer has `places_levels` (a TopoPlacer created
        with level_placement=True, whose snapshot holds the partitions of set_exclusive_levels), and its
        exclusive_domain is a domain of that level.  In a committed batch this also needs `places_committed_levels`
        (a TopoPlacer created with committed_levels=True).  Otherwise such a group gets no hint and a logged reason
        (no_hint[(ns, name)]): a hint into a domain of the wrong key is worse than none.
        alternates: next-best nodes per replica carried beside the hint (DESIGN.md §3.10, at most 8).  0 keeps the
        single-node hint; with n > 0 the snapshot call is rbgtopo_place_groups_ranked, which places identically and
        also ranks, per replica, the nodes that still have room once its group is placed.  A committed batch of
        one-pod replicas goes through rbgtopo_place_groups_committed_ranked (§3.14) when the placer has
        `places_committed_ranked`: same hints as rbgtopo_place_groups_committed, and alternates that still have
        room, and meet no exclusive claim of another gid, once the whole batch is placed.  A placer without it gives
        committed hints without alternates.  A committed batch placed through rbgtopo_place_groups_lw_committed
        (below) gets alternates from rbgtopo_place_groups_lw_committed_ranked (§3.15) when the placer has
        `places_lw_committed_ranked`, for its one-pod and its multi-pod groups alike; a placer without it gives that
        batch's hints without alternates.
        On a placer with world > 1 (node-axis shards) that has `places_sharded_ranked`, the snapshot call and the
        committed one-pod call with alternates are their sharded forms, place_groups_ranked_sharded and
        place_groups_committed_ranked_sharded (§3.17): every rank's manager must reconcile the same groups, and gets
        the hints and alternates of a world = 1 placer.  all_gather(ptr, nbytes) is their collective (None: the
        placer's default, torch.distributed over the initialised process group).  Leader-worker groups and committed
        leader-worker batches on a placer with world > 1 that has `places_lw_sharded` (a TopoPlacer created with
        lw_shards=True, §3.18) go through place_groups_lw / place_groups_lw_committed, and with alternates through
        place_groups_lw_ranked_sharded / place_groups_lw_committed_ranked_sharded over the same all_gather: the hints
        and alternates of a world = 1 placer, keyed by pod name.  Without it they are routed as at world = 1.
        leader_worker: a group with a role of lws_size > 1 is placed through rbgtopo_place_groups_lw (DESIGN.md
        §3.11): every replica of such a role is lws_size pods, placed all or nothing, and the hints are keyed by pod
        name, "{rbg}-{role}-{ordinal}-{k}" (k = 0 the leader); standalone roles keep "{rbg}-{role}-{ordinal}".  A
        role annotation COLOCATE_KEY names the topology key whose one domain must hold all pods of a replica; it
        resolves against exclusive_keys like an exclusive key (None: the level-0 label).  An unknown key, a level
        the snapshot does not hold leave such a group without a hint and log why.  A committed batch with such a
        group and no group at an exclusive level >= 1 goes through ONE rbgtopo_place_groups_lw_committed call (§3.13)
        when the placer has `places_lw_committed`: standalone groups take (1, -1) for every role and keep their RoleID
        keys.  Groups at exclusive levels >= 1 may be in that batch too when the placer also has
        `places_lw_committed_levels` (a TopoPlacer created with lw_committed_levels=True, §3.16).  Otherwise (levels
        >= 1 without it, or a placer without `places_lw_committed`) such a group gets no hint and a logged reason.  With
        alternates, such a group is placed through rbgtopo_place_groups_lw_ranked (§3.12) when the placer has
        `places_lw_ranked`, and its alternates are keyed by pod name and stay inside each replica's co-location
        domain; a placer without it gives no hint for such a group.
        False (default): those groups are placed as before, one pod per replica.
        node_classes: the classes installed on the placer (ingest.build_node_classes, then
        placer.set_node_classes(node_classes.node_class, node_classes.n_classes)); DESIGN.md §3.19.  A group with a role
        whose pod template excludes an installed class (ingest.role_admit over its nodeSelector, required node
        affinity and tolerations) is placed through rbgtopo_place_groups_eligible (_ranked with alternates), a
        leader-worker group with its (S, C) table and pod-keyed hints, so no hint or alternate lands on a node the role
        cannot run on.  A committed batch holding such a group goes through rbgtopo_place_groups_eligible_committed
        (§3.20) on a placer with `places_eligible_committed` (see reconcile_pod_groups).  Such a group gets no hint and
        a logged reason in a committed batch on a placer without that call or whose levels it cannot place, on a
        placer with world > 1 or without `places_eligible`, on the step-batch path, and so does a group whose
        selector the classes cannot decide.  Every other group is placed exactly as without node_classes.  None
        (default): eligibility is not looked at."""
        if not 0 <= alternates <= 8:
            raise ValueError(f"alternates must be in [0, 8], got {alternates}")
        self.alternates = int(alternates)
        self.placer = placer
        self.arith = HostArith()
        self.inner = inner
        self.exclusive_keys = None if exclusive_keys is None else tuple(exclusive_keys)
        self.leader_worker = bool(leader_worker)
        self.all_gather = all_gather
        self.no_hint: Dict[Tuple[str, str], str] = {}
        self._hints: Dict[Tuple[str, str], Placement] = {}
        self.node_classes = node_classes

    def exclusive_level(self, rbg: RoleBasedGroup, committed: bool = False) -> Tuple[int, str]:
        """(level of the group's exclusive key, reason for no hint or "")."""
        key = rbg.annotations.get(EXCLUSIVE_TOPOLOGY_KEY)
        if key is None or self.exclusive_keys is None:
            return 0, ""
        if key not in self.exclusive_keys:
            return -1, f"exclusive key {key!r} is not configured"
        lv = self.exclusive_keys.index(key)
        if lv == 0:
            return 0, ""
        if not getattr(self.placer, "places_levels", False):
            return lv, f"exclusive key {key!r} is not the level-0 label: no placement at that level yet"
        if committed and not getattr(self.placer, "places_committed_levels", False):
            return lv, f"exclusive key {key!r} is not the level-0 label: committed batches place level 0 only"
        return lv, ""

    def lw_committed(self, rbgs: Sequence[RoleBasedGroup], committed: bool) -> bool:
        """A committed batch placed by one rbgtopo_place_groups_lw_committed call: it has a leader-worker group, the
        placer places such batches, and it has no group at an exclusive level >= 1 unless the placer places those in
        such batches too (`places_lw_committed_levels`)."""
        return (committed and getattr(self.placer, "places_lw_committed", False)
                and any(self.is_leader_worker(r) for r in rbgs)
                and (getattr(self.placer, "places_lw_committed_levels", False)
                     or not any(self.exclusive_level(r, True)[0] > 0 for r in rbgs)))

    def eligible_committed(self, rbgs: Sequence[RoleBasedGroup], committed: bool) -> bool:
        """A committed batch placed by one rbgtopo_place_groups_eligible_committed call (DESIGN.md §3.20): it holds a
        restricted group that gets a hint (its selectors decided, its exclusive key placeable), the placer places
        such batches (`places_eligible_committed`, world == 1), and it has no group at an exclusive level >= 1 unless
        the placer places those in committed leader-worker batches (`places_lw_committed_levels`), as lw_committed."""
        return (committed and getattr(self.placer, "places_eligible_committed", False)
                and getattr(self.placer, "world", 1) == 1
                and any(self.is_restricted(r) and not self.role_masks(r)[1] and not self.exclusive_level(r, True)[1]
                        for r in rbgs)
                and (getattr(self.placer, "places_lw_committed_levels", False)
                     or not any(self.exclusive_level(r, True)[0] > 0 for r in rbgs)))

    def role_masks(self, rbg: RoleBasedGroup) -> Tuple[List[int], str]:
        """(class mask per role in spec order, reason for no hint or "") under node_classes (DESIGN.md §3.19)."""
        try:
            return [role_admit(self.node_classes, r.node_selector, r.node_affinity, r.tolerations)
                    for r in rbg.roles], ""
        except NotDecidable as e:
            return [], f"node eligibility: {e}"

    def is_restricted(self, rbg: RoleBasedGroup) -> bool:
        """A role's pod template excludes an installed node class (or cannot be decided per class): the group is
        placed by rbgtopo_place_groups_eligible, or gets no hint."""
        if self.node_classes is None:
            return False
        masks, reason = self.role_masks(rbg)
        full = (1 << self.node_classes.n_classes) - 1
        return bool(reason) or any(m & full != full for m in masks)

    def _eligibility_reason(self, rbg: RoleBasedGroup, committed: bool, waves: bool, elig_commit: bool = False) -> str:
        """Why a restricted group gets no hint, or "".  elig_commit: the committed batch goes through
        rbgtopo_place_groups_eligible_committed (eligible_committed)."""
        if not self.is_restricted(rbg):
            return ""
        reason = self.role_masks(rbg)[1]
        if reason:
            return reason
        if committed and not elig_commit:
            return "node eligibility: committed batches place no node classes"
        if waves:
            return "node eligibility: the step-batch path places no node classes"
        if getattr(self.placer, "world", 1) > 1:
            return "node eligibility: placers with world > 1 place no node classes"
        if not getattr(self.placer, "places_eligible", False):
            return "node eligibility: the placer has no rbgtopo_place_groups_eligible"
        return ""

    def _split_no_hint(self, rbgs: Sequence[RoleBasedGroup], committed: bool = False, waves: bool = False):
        """The groups that get a hint, and a no-hint Placement per group that does not (logged, hint dropped)."""
        keep, skipped = [], {}
        elig_commit = not waves and self.eligible_committed(rbgs, committed)
        lw_commit = elig_commit or self.lw_committed(rbgs, committed)
        for i, r in enumerate(rbgs):
            _, reason = self.exclusive_level(r, committed)
            if not reason:
                reason = self._eligibility_reason(r, committed, waves, elig_commit)
            if not reason and (self.is_restricted(r) or elig_commit):   # the eligible calls rank for every group
                if self.is_leader_worker(r):
                    reason = self.role_pods(r)[1]
            elif not reason and self.is_leader_worker(r):
                if committed and not lw_commit:
                    reason = "leader-worker replicas: committed batches place one pod per replica"
                elif self.alternates and not getattr(self.placer, "places_lw_ranked", False):
                    reason = "leader-worker replicas: no ranked alternates for them"
                else:
                    reason = self.role_pods(r)[1]
            if not reason:
                keep.append(r)
                continue
            self._hints.pop((r.namespace, r.name), None)
            self.no_hint[(r.namespace, r.name)] = reason
            logging.getLogger(__name__).info("no placement hint for %s/%s: %s", r.namespace, r.name, reason)
            skipped[i] = Placement(RBGTOPO_NO_HINT, {}, -1, 0)
        return keep, skipped

    def _lw_sharded(self) -> bool:
        """Leader-worker calls on node-axis shards (§3.18): a placer with world > 1 that places them there."""
        return getattr(self.placer, "world", 1) > 1 and getattr(self.placer, "places_lw_sharded", False)

    def is_leader_worker(self, rbg: RoleBasedGroup) -> bool:
        """Placed through rbgtopo_place_groups_lw: the manager was asked to and a role runs multi-pod replicas."""
        return self.leader_worker and any(r.lws_size > 1 for r in rbg.roles)

    def role_pods(self, rbg: RoleBasedGroup) -> Tuple[List[Tuple[int, int]], str]:
        """((pods per replica S, co-location level C) per role in spec order, reason for no hint or "")."""
        out = []
        for r in rbg.roles:
            key, level = r.annotations.get(COLOCATE_KEY), -1
            if key is not None:
                if self.exclusive_keys is None:
                    level = 0
                elif key not in self.exclusive_keys:
                    return [], f"co-location key {key!r} of role {r.name} is not configured"
                else:
                    level = self.exclusive_keys.index(key)
                    if level > getattr(self.placer, "_n_levels", 0):
                        return [], f"co-location key {key!r} of role {r.name}: the snapshot holds no level {level}"
            out.append((max(1, r.lws_size), level))
        return out, ""

    @staticmethod
    def _merge(rbgs, placed, skipped):
        it = iter(placed)
        return [skipped[i] if i in skipped else next(it) for i in range(len(rbgs))]

    # -- ReconcilePodGroup(ctx, rbg, ...) for one group -------------------------
    def ReconcilePodGroup(self, rbg: RoleBasedGroup) -> Placement:  # noqa: N802 (reference name)
        return self.reconcile_pod_groups([rbg])[0]

    # -- batched form: the concurrent reconciles of one informer snapshot
    #    (cmd/rbgs/main.go:140-143) coalesced into level-synchronous launches.
    #    The level/wave loop runs behind the ABI (rbgtopo_place_groups, C++).
    def groups_blob(self, rbgs: Sequence[RoleBasedGroup]):
        """Marshal RoleBasedGroups into the GROUPS wire format (the Go shim does
        the same from the typed objects).  Returns (blob, runs)."""
        runs = [_GroupRun(r, self.arith, plan_waves=False, excl_level=self.exclusive_level(r)[0]) for r in rbgs]
        gb = GroupsBuilder()
        for g in runs:
            roles = [(g.level_of[ri], g.pending[ri], g.rbg.roles[ri].demand,
                      ROLE_EXCLUSIVE if g.role_excl[ri] else 0) for ri in g.order]
            pair = [[int(g.pair[a, b]) for b in g.order] for a in g.order]
            pos = {ri: k for k, ri in enumerate(g.order)}
            anchors = [(n, pos[q], c) for (n, q), c in sorted(g.anchors.items())]
            flags = (STEP_EXCLUSIVE if g.exclusive else 0) | (STEP_GANG if g.gang else 0)
            gb.add(Group(gid=g.rbg.gid, roles=roles, pair=pair, anchors=anchors, flags=flags,
                         fixed_domain=g.fixed_domain if g.exclusive else -1, level=g.excl_level))
        return gb.build(), runs

    def reconcile_pod_groups(self, rbgs: Sequence[RoleBasedGroup], committed: bool = False) -> List[Placement]:
        """committed=False: every group against the same snapshot (DESIGN.md §3.7), like concurrent reconciles.
        committed=True: a committed batch (§3.8) in the order given — each group sees the capacity and exclusive
        domains the groups before it took, so the hints of one call never contradict each other (the controller
        passes the groups ordered by namespaced name).  With alternates, a committed batch of one-pod replicas gets
        them from place_groups_committed_ranked (§3.14) when the placer has `places_committed_ranked`: room and
        exclusive claims counted after the whole batch.  A committed batch with leader-worker groups gets them from
        place_groups_lw_committed_ranked (§3.15) when the placer has `places_lw_committed_ranked`.  A committed batch
        that holds a group restricted by node_classes goes through ONE place_groups_eligible_committed call (_ranked
        with alternates, §3.20) when the placer has `places_eligible_committed` and every group's level is placeable
        (as for lw_committed): every role carries its class mask (all ones for unrestricted groups), role_pods is
        given only when a leader-worker group is in the batch, and the hints of leader-worker groups are keyed by pod
        name.  The restricted groups' claims then count for the groups after them too."""
        all_rbgs = rbgs
        elig_commit = self.eligible_committed(rbgs, committed)
        lw_commit = self.lw_committed(rbgs, committed)
        rbgs, skipped = self._split_no_hint(rbgs, committed)
        if not rbgs:
            return self._merge(all_rbgs, [], skipped)
        if elig_commit:   # one call in the given order, with node eligibility for every role
            blob, runs = self.groups_blob(rbgs)
            masks = [self.role_masks(g.rbg)[0] if self.is_restricted(g.rbg) else [ALL_CLASSES] * len(g.rbg.roles)
                     for g in runs]
            role_admit_ = [masks[k][ri] for k, g in enumerate(runs) for ri in g.order]
            pods = None
            if any(self.is_leader_worker(g.rbg) for g in runs):
                pods = [self.role_pods(g.rbg)[0] if self.is_leader_worker(g.rbg) else [(1, -1)] * len(g.rbg.roles)
                        for g in runs]
            role_pods = None if pods is None else [pods[k][ri] for k, g in enumerate(runs) for ri in g.order]
            alt_node = None
            if self.alternates > 0:
                assign, status, domain, _, _, alt_node, _ = self.placer.place_groups_eligible_committed_ranked(
                    blob, role_pods, role_admit_, self.alternates)
            else:
                assign, status, domain, _ = self.placer.place_groups_eligible_committed(blob, role_pods, role_admit_)
            return self._merge(all_rbgs, self._placements(runs, assign, status, domain, alt_node, pods), skipped)
        if lw_commit:   # one call in the given order: every group sees what the groups before it took
            blob, runs = self.groups_blob(rbgs)
            pods = [self.role_pods(g.rbg)[0] if self.is_leader_worker(g.rbg) else [(1, -1)] * len(g.rbg.roles)
                    for g in runs]
            role_pods = [pods[k][ri] for k, g in enumerate(runs) for ri in g.order]
            alt_node = None
            if self.alternates > 0 and self._lw_sharded():
                assign, status, domain, _, _, alt_node, _ = self.placer.place_groups_lw_committed_ranked_sharded(
                    blob, role_pods, self.alternates, self.all_gather)
            elif self.alternates > 0 and getattr(self.placer, "places_lw_committed_ranked", False):
                assign, status, domain, _, _, alt_node, _ = self.placer.place_groups_lw_committed_ranked(
                    blob, role_pods, self.alternates)
            else:
                assign, status, domain, _ = self.placer.place_groups_lw_committed(blob, role_pods)
            return self._merge(all_rbgs, self._placements(runs, assign, status, domain, alt_node, pods), skipped)
        elig = [i for i, r in enumerate(rbgs) if self.is_restricted(r)]
        lw = [i for i, r in enumerate(rbgs) if self.is_leader_worker(r) and i not in elig]
        plain = [i for i, r in enumerate(rbgs) if not self.is_leader_worker(r) and i not in elig]
        done: List[Optional[Placement]] = [None] * len(rbgs)   # by position in rbgs
        if elig:   # DESIGN.md §3.19: masks in blob order, (S, C) when a leader-worker group is among them
            blob, runs = self.groups_blob([rbgs[i] for i in elig])
            masks = [self.role_masks(g.rbg)[0] for g in runs]
            role_admit_ = [masks[k][ri] for k, g in enumerate(runs) for ri in g.order]
            pods = None
            if any(self.is_leader_worker(g.rbg) for g in runs):
                pods = [self.role_pods(g.rbg)[0] if self.is_leader_worker(g.rbg) else [(1, -1)] * len(g.rbg.roles)
                        for g in runs]
            role_pods = None if pods is None else [pods[k][ri] for k, g in enumerate(runs) for ri in g.order]
            alt_node = None
            if self.alternates > 0:
                assign, status, domain, _, alt_node, _ = self.placer.place_groups_eligible_ranked(
                    blob, role_pods, role_admit_, self.alternates)
            else:
                assign, status, domain = self.placer.place_groups_eligible(blob, role_pods, role_admit_)
            for i, p in zip(elig, self._placements(runs, assign, status, domain, alt_node, pods)):
                done[i] = p
        if plain:
            blob, runs = self.groups_blob([rbgs[i] for i in plain])
            alt_node = None
            sharded = getattr(self.placer, "world", 1) > 1 and getattr(self.placer, "places_sharded_ranked", False)
            if committed and self.alternates > 0 and sharded:
                assign, status, domain, _, _, alt_node, _ = self.placer.place_groups_committed_ranked_sharded(
                    blob, self.alternates, self.all_gather)
            elif committed and self.alternates > 0 and getattr(self.placer, "places_committed_ranked", False):
                assign, status, domain, _, _, alt_node, _ = self.placer.place_groups_committed_ranked(
                    blob, self.alternates)
            elif committed:
                assign, status, domain, _ = self.placer.place_groups_committed(blob)
            elif self.alternates > 0 and sharded:
                assign, status, domain, _, alt_node, _ = self.placer.place_groups_ranked_sharded(
                    blob, self.alternates, self.all_gather)
            elif self.alternates > 0:
                assign, status, domain, _, alt_node, _ = self.placer.place_groups_ranked(blob, self.alternates)
            else:
                assign, status, domain = self.placer.place_groups(blob)
            for i, p in zip(plain, self._placements(runs, assign, status, domain, alt_node, None)):
                done[i] = p
        if lw:
            blob, runs = self.groups_blob([rbgs[i] for i in lw])
            pods = [self.role_pods(g.rbg)[0] for g in runs]
            role_pods = [pods[k][ri] for k, g in enumerate(runs) for ri in g.order]
            alt_node = None
            if self.alternates > 0 and self._lw_sharded():
                assign, status, domain, _, alt_node, _ = self.placer.place_groups_lw_ranked_sharded(
                    blob, role_pods, self.alternates, self.all_gather)
            elif self.alternates > 0:
                assign, status, domain, _, alt_node, _ = self.placer.place_groups_lw_ranked(blob, role_pods,
                                                                                           self.alternates)
            else:
                assign, status, domain = self.placer.place_groups_lw(blob, role_pods)
            for i, p in zip(lw, self._placements(runs, assign, status, domain, alt_node, pods)):
                done[i] = p
        return self._merge(all_rbgs, done, skipped)

    def _placements(self, runs, assign, status, domain, alt_node, pods) -> List[Placement]:
        """Per group: the hints of one placement call.  pods: (S, C) per role of every group (leader-worker call) —
        a role with S > 1 gets one key per pod, "{rbg}-{role}-{ordinal}-{k}" — or None (one pod per replica)."""
        out, off = [], 0
        n_nodes = self.placer.n_nodes
        for i, g in enumerate(runs):
            nodes: Dict[str, int] = {}
            alts: Dict[str, List[int]] = {}
            for ri in g.order:
                role = g.rbg.roles[ri]
                S = 1 if pods is None else pods[i][ri][0]
                for c in range(g.pending[ri]):
                    key = f"{g.rbg.name}-{role.name}-{g.first_ordinal[ri] + c}"
                    for k in range(S):
                        pod = key if S == 1 else f"{key}-{k}"
                        nodes[pod] = int(assign[off])
                        if alt_node is not None:
                            alts[pod] = [int(x) for x in alt_node[off] if x >= 0]
                        off += 1
            p = Placement(int(status[i]), nodes, int(domain[i]), len(nodes) * n_nodes, alts)
            self._hints[(g.rbg.namespace, g.rbg.name)] = p
            out.append(p)
        return out

    # -- the same loop in Python over single-level batches (rbgtopo_score_assign):
    #    kept as the readable mirror of the C++ loop and for cross-checks.
    def reconcile_pod_groups_by_waves(self, rbgs: Sequence[RoleBasedGroup]) -> List[Placement]:
        all_rbgs = rbgs
        rbgs, skipped = self._split_no_hint(rbgs, waves=True)
        runs = [_GroupRun(r, self.arith, excl_level=self.exclusive_level(r)[0]) for r in rbgs]
        n_nodes = self.placer.n_nodes
        w = 0
        while True:
            active = [g for g in runs if not g.failed and w < len(g.waves)]
            if not active:
                break
            bb = BlobBuilder()
            for g in active:
                bb.add(g.step(w))
            blob = bb.build()
            assign, status, domain = self.placer.score_assign(blob)
            off = 0
            for i, g in enumerate(active):
                r = g.waves[w]
                cnt = sum(c for _, _, c in r.roles)
                g.absorb(w, assign[off:off + cnt], int(status[i]), int(domain[i]), n_nodes)
                off += cnt
            w += 1
        out = []
        for g in runs:
            nodes = {}
            for wv in g.waves:   # every pending replica, in (level, name, ordinal) order
                for ri, ordinal, cnt in wv.roles:
                    for c in range(cnt):
                        key = f"{g.rbg.name}-{g.rbg.roles[ri].name}-{ordinal + c}"
                        nodes[key] = -1 if g.failed else g.result_nodes.get(key, -1)
            if g.failed:   # gang: all-or-nothing over GetGroupSize() pods (manager.go:131)
                p = Placement(2, nodes, -1, g.scores)
            else:
                p = Placement(g.status, nodes, g.fixed_domain if g.exclusive else -1, g.scores)
            self._hints[(g.rbg.namespace, g.rbg.name)] = p
            out.append(p)
        return self._merge(all_rbgs, out, skipped)

    # -- coordination-aware batching (SURVEY.md §8f rank 4) ------------------------
    def coordination_batches(self, rbg: RoleBasedGroup, max_batches: int = 64) -> List[Dict[str, int]]:
        """The sequence of scaling targets the controller will go through if every batch it
        creates gets scheduled and ready: the reference paces a group in MaxSkew-bounded steps
        (scaler.go:70-172), one step per reconcile.  Returned without touching `rbg`."""
        st = {r.name: RoleStatus(**vars(rbg.status.get(r.name, RoleStatus()))) for r in rbg.roles}
        out: List[Dict[str, int]] = []
        for _ in range(max_batches):
            probe = RoleBasedGroup(rbg.namespace, rbg.name, rbg.roles, scaling_rules=rbg.scaling_rules, status=st)
            tgt = self.arith.scaling_targets(probe)
            if tgt is None or all(tgt.get(nm, s.replicas) <= s.replicas for nm, s in st.items()):
                break
            out.append(tgt)
            for nm, t in tgt.items():
                st[nm] = RoleStatus(replicas=t, ready=t, scheduled=t)
        return out

    def reconcile_ahead(self, rbg: RoleBasedGroup, batches: int = 2, by_waves: bool = False) -> List[Placement]:
        """Place the current coordination batch and pre-place the next `batches - 1` in ONE pass:
        the group is placed up to the targets of the last of those batches (levels and waves keep
        the capacity consistent across them), and the result is split by ordinal — replica
        `ordinal` of a role belongs to the first batch whose target exceeds it — so the hints of
        the coming batches exist before the controller asks for them."""
        tg = self.coordination_batches(rbg, batches)
        if not tg:
            return []
        cur = {r.name: rbg.current.get(r.name, rbg.status[r.name].replicas if r.name in rbg.status else 0)
               for r in rbg.roles}
        step = RoleBasedGroup(rbg.namespace, rbg.name, rbg.roles, annotations=rbg.annotations, gid=rbg.gid,
                              policy_rules=rbg.policy_rules, targets=tg[-1], current=cur, placed=rbg.placed,
                              exclusive_domain=rbg.exclusive_domain)
        p = (self.reconcile_pod_groups_by_waves if by_waves else self.reconcile_pod_groups)([step])[0]
        out = [Placement(p.status, {}, p.domain, 0) for _ in tg]
        names = sorted((r.name for r in rbg.roles), key=len, reverse=True)
        spec_replicas = {r.name: r.replicas for r in rbg.roles}
        n_nodes = self.placer.n_nodes
        for key, node in p.nodes.items():
            stem, ordinal = key[len(rbg.name) + 1:key.rfind("-")], int(key[key.rfind("-") + 1:])
            role = next(nm for nm in names if nm == stem)
            # a role no ScalingRule paces is created whole by the current reconcile (its target is the
            # spec's replica count in every batch): its replicas belong to batch 0
            k = next((i for i, t in enumerate(tg) if ordinal < t.get(role, spec_replicas[role])), 0)
            out[k].nodes[key] = node
            out[k].scores += n_nodes
        return out

    # -- InjectPodGroupLabels(rbg, podTemplateSpec) ------------------------------
    def InjectPodGroupLabels(self, rbg: RoleBasedGroup, pod_template: dict) -> None:  # noqa: N802
        """Adds the serialized RoleID -> node map as a pod-template annotation
        (the template is per role, not per replica: SURVEY.md §8b "Injection")."""
        meta = pod_template.setdefault("metadata", {})
        if rbg.annotations.get(GANG_SCHEDULING_KEY) == "true":     # the wrapped plugin's injection, unchanged
            if self.inner == "scheduler-plugins":
                meta.setdefault("labels", {})[KUBE_POD_GROUP_LABEL] = rbg.name
            elif self.inner == "volcano":
                meta.setdefault("annotations", {})[VOLCANO_GROUP_ANNOTATION] = rbg.name
        p = self._hints.get((rbg.namespace, rbg.name))
        if p is None:
            return
        ann = meta.setdefault("annotations", {})
        ann[PLACEMENT_HINT_KEY] = json.dumps({k: v for k, v in sorted(p.nodes.items()) if v >= 0},
                                             separators=(",", ":"))
        alts = {k: v for k, v in sorted(p.alternates.items()) if v}
        if alts:
            ann[PLACEMENT_ALTERNATES_KEY] = json.dumps(alts, separators=(",", ":"))


def new_pod_group_manager(scheduler_name: str, placer: TopoPlacer) -> B200TopoPodGroupManager:
    """The case added to NewPodGroupManager (pkg/scheduler/podgroup_manager.go:82-92)."""
    if scheduler_name != SCHEDULER_PLUGIN_NAME:
        raise ValueError(f'unsupported scheduler-name "{scheduler_name}": this mirror only provides '
                         f'"{SCHEDULER_PLUGIN_NAME}"')
    return B200TopoPodGroupManager(placer)
