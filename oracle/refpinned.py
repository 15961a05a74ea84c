"""CPU ORACLE — reference-pinned arithmetic (SURVEY.md §8a rows a6-a15).

TEST INFRASTRUCTURE ONLY: imported by tests/ (and nothing under rbg_b200/).
Each function restates one Go function of sgl-project/rbg and cites it
(paths relative to the reference checkout).  These are O(#roles) scalar functions, so
plain Python is the right tool; Python ``float`` is IEEE-754 binary64 == Go
``float64`` and ``math.ceil/floor`` == ``math.Ceil/Floor``.  They are pinned by
tests/test_refpinned_golden.py against every table the reference's own tests
hold for them (SURVEY.md Appendix B, transcribed into tests/golden/*.json).
"""
from __future__ import annotations

import hashlib
import math
from typing import Dict, List, Optional, Sequence, Tuple

ORDER_SCHEDULED = "OrderScheduled"  # api/workloads/v1alpha2/coordinatedpolicy_types.go
ORDER_READY = "OrderReady"


class RefError(Exception):
    """Stands for a non-nil Go ``error`` return."""


# --------------------------------------------------------------------------
# vendor/k8s.io/apimachinery/pkg/util/intstr/intstr.go
# --------------------------------------------------------------------------
IntOrStr = object  # int (Type==Int) or str (Type==String)


def _atoi(s: str) -> int:
    """strconv.Atoi: optional sign, decimal digits only."""
    t = s
    if t[:1] in "+-":
        t = t[1:]
    if not t or not all("0" <= ch <= "9" for ch in t):
        raise RefError(f"invalid value {s!r}")
    return int(s)


def get_int_or_percent_value_safely(v) -> Tuple[int, bool]:
    """getIntOrPercentValueSafely, intstr.go:238-258."""
    if isinstance(v, bool):
        raise RefError("invalid type: neither int nor percentage")
    if isinstance(v, int):
        return v, False
    if isinstance(v, str):
        if not v.endswith("%"):
            raise RefError("invalid type: string is not a percentage")
        return _atoi(v[:-1]), True
    raise RefError("invalid type: neither int nor percentage")


def get_scaled_value_from_int_or_percent(v, total: int, round_up: bool) -> int:
    """GetScaledValueFromIntOrPercent, intstr.go:181-197."""
    if v is None:
        raise RefError("nil value for IntOrString")
    value, is_percent = get_int_or_percent_value_safely(v)
    if is_percent:
        x = float(value) * float(total) / 100
        value = int(math.ceil(x)) if round_up else int(math.floor(x))
    return value


# --------------------------------------------------------------------------
# pkg/utils/utils.go
# --------------------------------------------------------------------------
def calculate_partition_replicas(partition, replicas: Optional[int]) -> int:
    """CalculatePartitionReplicas, pkg/utils/utils.go:139-162."""
    if partition is None:
        return 0
    reps = 1 if replicas is None else int(replicas)
    p = get_scaled_value_from_int_or_percent(partition, reps, True)
    if reps >= 1 and p == reps and isinstance(partition, str) and partition != "100%":
        p = reps - 1
    return max(min(p, reps), 0)


def parse_intstr_as_non_zero(p, replicas: int) -> Tuple[int, Optional[str]]:
    """ParseIntStrAsNonZero, pkg/utils/utils.go:177-185 -> (value, err)."""
    try:
        value = get_scaled_value_from_int_or_percent(p, int(replicas), True)
    except RefError as e:
        return 1, str(e)
    return (1 if value < 1 else value), None


def abs_float64(x: float) -> float:
    """ABSFloat64, pkg/utils/utils.go:187-192."""
    return -x if x < 0 else x


# --------------------------------------------------------------------------
# pkg/coordination/coordinationscaling/scaler.go
# --------------------------------------------------------------------------
def parse_percentage(s: str) -> float:
    """parsePercentage, scaler.go:253-270."""
    s = s.strip()  # strings.TrimSpace
    if not s.endswith("%"):
        raise RefError("percentage string must end with '%'")
    num_str = s[:-1]
    try:
        if num_str.strip() != num_str or "_" in num_str or not num_str:
            raise ValueError(num_str)
        num = float(num_str)  # strconv.ParseFloat(numStr, 64)
    except ValueError as e:
        raise RefError(f"failed to parse percentage number: {e}") from None
    if num < 0 or num > 100:
        raise RefError(f"percentage must be between 0 and 100, got {num}")
    return num / 100.0


def new_coordination_scaler(policy_rule: Optional[dict]) -> Tuple[float, dict]:
    """NewCoordinationScalerFromPolicy, scaler.go:44-65.

    policy_rule: {"roles": [...], "scaling": None | {"maxSkew": str|None,
    "progression": str|None}} -> (maxSkew, rule)."""
    if policy_rule is None or policy_rule.get("scaling") is None:
        raise RefError("invalid policy configuration: scaling strategy is nil")
    ms = policy_rule["scaling"].get("maxSkew")
    max_skew_str = "100%" if ms is None else str(ms)
    try:
        return parse_percentage(max_skew_str), policy_rule
    except RefError as e:
        raise RefError(f"failed to parse maxSkew: {e}") from None


def can_proceed_to_next_batch(roles: Sequence[str], states: Dict[str, dict],
                              progression: str) -> bool:
    """canProceedToNextBatch, scaler.go:192-242."""
    if all(states[r]["current"] >= states[r]["desired"] for r in roles):
        return True
    for r in roles:
        st = states[r]
        if st["current"] >= st["desired"]:
            continue
        if st["current"] == 0:
            continue
        # Go `switch progression`: the zero value "" matches neither case, so an
        # unset Progression gates nothing (getProgressionType's OrderScheduled
        # default, scaler.go:183-188, only applies when the rule itself is nil).
        if progression == ORDER_SCHEDULED:
            if st["scheduled"] < st["current"]:
                return False
        elif progression == ORDER_READY:
            if st["ready"] < st["current"]:
                return False
    return True


def calculate_target_replicas(max_skew: float, roles: Sequence[str],
                              states: Dict[str, dict],
                              progression: str = "") -> Dict[str, int]:
    """CoordinationScaler.CalculateTargetReplicas, scaler.go:70-172.

    states[role] = {"desired","current","scheduled","ready"} (int32)."""
    if len(states) == 0:
        raise RefError("no role states provided")
    for r in roles:
        if r not in states:
            raise RefError(f"role {r} not found in roleStates")
    if not can_proceed_to_next_batch(roles, states, progression):
        return {r: states[r]["current"] for r in roles}
    prog = []
    for r in roles:
        st = states[r]
        if st["desired"] == 0:
            p = 1.0 if st["current"] == 0 else 0.0
        else:
            p = float(st["current"]) / float(st["desired"])
        prog.append((r, st["desired"], st["current"], p))
    # sort.Slice ascending by progress (unstable in Go; ties give the same
    # minProgress so the outcome does not depend on their order)
    prog.sort(key=lambda x: x[3])
    min_progress = prog[0][3]
    for _, desired, current, p in prog:
        if current < desired:
            min_progress = p
            break
    max_allowed = min_progress + max_skew
    out: Dict[str, int] = {}
    for r, desired, current, p in prog:
        if current >= desired:
            out[r] = desired
            continue
        if p >= max_allowed:
            out[r] = current
            continue
        target = int(math.ceil(max_allowed * float(desired)))
        if target > desired:
            target = desired
        if target <= current and current < desired:
            target = current + 1
        out[r] = target
    return out


# --------------------------------------------------------------------------
# internal/controller/workloads/rolebasedgroup_controller.go
# --------------------------------------------------------------------------
def calculate_scaling_for_all_coordination(policy_rules: Sequence[dict],
                                           desired: Dict[str, int],
                                           statuses: Dict[str, dict],
                                           scheduled: Dict[str, int]) -> Dict[str, int]:
    """CalculateScalingForAllCoordination, rolebasedgroup_controller.go:968-1054.

    desired[role] = spec replicas (GetRoleReplicasV2, pkg/utils/utils.go:165-175);
    statuses[role] = {"replicas","ready"}; scheduled[role] = pods with a nodeName
    (getScheduledReplicas, :1057-1080)."""
    result: Dict[str, int] = {}
    processed = set()
    for rule in policy_rules:
        if rule.get("scaling") is None:
            continue
        max_skew, _ = new_coordination_scaler(rule)
        states = {}
        for r in rule["roles"]:
            st = statuses.get(r, {})
            states[r] = {"desired": desired.get(r, 0), "current": st.get("replicas", 0),
                         "ready": st.get("ready", 0), "scheduled": scheduled.get(r, 0)}
        targets = calculate_target_replicas(max_skew, rule["roles"], states,
                                            rule["scaling"].get("progression") or "")
        for r, t in targets.items():
            if r in processed:
                if t < result[r]:
                    result[r] = t
            else:
                result[r] = t
                processed.add(r)
    return result


def _go_round(x: float) -> float:
    """math.Round: half away from zero."""
    return math.floor(x + 0.5) if x >= 0 else -math.floor(-x + 0.5)


def calculate_coordination_updated_replicas_bound(max_skew, ref_updated: int,
                                                  ref_desired: int,
                                                  request_desired: int) -> Tuple[int, int]:
    """calculateCoordinationUpdatedReplicasBound, rolebasedgroup_controller.go:1328-1345."""
    if ref_desired == 0:
        return 0, 0
    try:
        s = get_scaled_value_from_int_or_percent(max_skew, 100, True)
    except RefError:
        s = 0  # the Go code drops the error; value is 0 then
    a, b, d = int(ref_updated), int(ref_desired), int(request_desired)
    lower = _go_round(float(max(100 * a * d - s * b * d, 0)) / float(100 * b))
    upper = _go_round(float(max(s * b * d + 100 * a * d, 0)) / float(100 * b))
    return int(lower), int(upper)


def get_fastest_and_slowest_role(roles: Sequence[str], desired: Dict[str, int],
                                 updated: Dict[str, int]) -> Tuple[str, str]:
    """getFastestAndSlowestRole, rolebasedgroup_controller.go:1265-1282.

    Go sorts an UnsortedList with an unstable sort; outcomes the reference
    tests pin do not depend on that.  We sort names first, then insertion-sort
    with the Go comparator, which is deterministic."""
    roles = sorted(set(roles))
    if len(roles) <= 1:
        return "", ""
    ratio = {}
    for r in roles:
        d = float(desired.get(r, 0))
        u = float(updated.get(r, 0))
        ratio[r] = (u / d) if d != 0 else (math.nan if u == 0 else math.inf)

    def less(a: str, b: str) -> bool:
        if abs_float64(ratio[a] - ratio[b]) > 1e-6:
            return ratio[a] < ratio[b]
        return desired.get(a, 0) > desired.get(b, 0)

    out: List[str] = []
    for r in roles:
        i = len(out)
        while i > 0 and less(r, out[i - 1]):
            i -= 1
        out.insert(i, r)
    return out[-1], out[0]


def calculate_next_rolling_target(max_skew_percent: str, roles: Sequence[str],
                                  desired: Dict[str, int], updated: Dict[str, int],
                                  ready: Dict[str, int]) -> Optional[Dict[str, int]]:
    """calculateNextRollingTarget, rolebasedgroup_controller.go:1223-1263."""
    fastest, slowest = get_fastest_and_slowest_role(roles, desired, updated)
    if fastest == "" or slowest == "":
        return None
    target = {r: updated.get(r, 0) for r in set(roles)}
    max_skew, _ = parse_intstr_as_non_zero(max_skew_percent, desired.get(slowest, 0))
    lower, upper = calculate_coordination_updated_replicas_bound(
        max_skew_percent, updated.get(fastest, 0), desired.get(fastest, 0),
        desired.get(slowest, 0))
    balance = (lower + upper + 1) >> 1
    dist = max(balance - updated.get(slowest, 0), 0)
    step = max(dist, max_skew >> 1)
    if ready.get(fastest, 0) == desired.get(fastest, 0):
        step = max(step, 1)
    target[slowest] = min(updated.get(slowest, 0) + step, upper + 1)
    return target


def merge_strategy_rolling_update(a: Dict[str, dict], b: Optional[Dict[str, dict]]) -> Dict[str, dict]:
    """mergeStrategyRollingUpdate, rolebasedgroup_controller.go:1284-1314.

    strategy = {"maxUnavailable": int|str|None, "partition": int|str|None}."""
    merged = {r: dict(s) for r, s in a.items()}
    for r, sb in (b or {}).items():
        if r not in merged:
            merged[r] = dict(sb)
            continue
        sa = merged[r]

        def scaled(v):
            try:
                return get_scaled_value_from_int_or_percent(v, 100, True)
            except RefError:
                return 0

        if scaled(sa.get("maxUnavailable")) > scaled(sb.get("maxUnavailable")):
            sa["maxUnavailable"] = sb.get("maxUnavailable")
        pa = scaled(sa["partition"]) if sa.get("partition") is not None else 0
        pb = scaled(sb["partition"]) if sb.get("partition") is not None else 0
        if pa < pb:
            sa["partition"] = sb.get("partition")
        merged[r] = sa
    return merged


# --------------------------------------------------------------------------
# pkg/dependency/dependency.go
# --------------------------------------------------------------------------
def dependency_order(dependencies: Dict[str, List[str]]) -> List[List[str]]:
    """dependencyOrder, pkg/dependency/dependency.go:129-205 (DFS levels; keys
    sorted first, so every level is lexicographic; cycle -> error)."""
    keys = sorted(dependencies)
    order = {k: -2 for k in keys}

    def visit(name: str) -> int:
        if order[name] >= 0:
            return order[name]
        if order[name] == -1:
            raise RefError(f"cycle detected for role '{name}'")
        order[name] = -1
        mx = 0
        for dep in dependencies[name]:
            if dep not in order:
                raise RefError(f"dependency '{dep}' not found for role '{name}'")
            mx = max(mx, visit(dep) + 1)
        order[name] = mx
        return mx

    for k in keys:
        if order[k] == -2:
            visit(k)
    levels: List[List[str]] = [[] for _ in range(max(order.values(), default=0) + 1)]
    for k in keys:
        levels[order[k]].append(k)
    return levels


# --------------------------------------------------------------------------
# api/workloads/v1alpha2/helper.go, pkg/scheduler/common, naming
# --------------------------------------------------------------------------
def get_group_size(roles: Sequence[dict]) -> int:
    """RoleBasedGroup.GetGroupSize, api/workloads/v1alpha2/helper.go:50-65.
    role = {"replicas": int, "lws": bool, "lws_size": int|None}."""
    ret = 0
    for role in roles:
        if role.get("lws"):
            size = role.get("lws_size")
            ret += (1 if size is None else int(size)) * int(role["replicas"])
        else:
            ret += int(role["replicas"])
    return ret


def get_workload_name(rbg_name: str, role_name: str) -> str:
    """GetWorkloadName, helper.go:68-81."""
    name = f"{rbg_name}-{role_name}"
    if len(name) > 63:
        name = name[:63].rstrip("-")
    return name


def gen_group_unique_key(namespace: str, name: str) -> str:
    """GenGroupUniqueKey, helper.go:135-144 (sha1 hex of "ns/name")."""
    return hashlib.sha1(f"{namespace}/{name}".encode()).hexdigest()


def inherit_pod_group_annotations(annotations: Optional[Dict[str, str]],
                                  *prefixes: str) -> Optional[Dict[str, str]]:
    """InheritPodGroupAnnotations, pkg/scheduler/common/annotation_inheritance.go:23-43."""
    if not annotations or not prefixes:
        return None
    out = {k: v for k, v in annotations.items() if any(k.startswith(p) for p in prefixes)}
    return out or None


def replica_name(set_name: str, ordinal: int) -> str:
    """pkg/reconciler/roleinstanceset/statefulmode/stateful_instance_set_utils.go:74-76."""
    return f"{set_name}-{ordinal}"


def exclusive_affinity_terms(unique_key: str, topology_key: str, affinity_key: str) -> dict:
    """setExclusiveAffinities, pkg/reconciler/pod_reconciler.go:172-231: the two
    required terms that define exclusive topology."""
    if not topology_key:
        raise RefError("topology key can't be nil")
    return {
        "podAffinity": {"topologyKey": topology_key,
                        "matchExpressions": [{"key": affinity_key, "operator": "In",
                                              "values": [unique_key]}]},
        "podAntiAffinity": {"topologyKey": topology_key,
                            "matchExpressions": [
                                {"key": affinity_key, "operator": "Exists"},
                                {"key": affinity_key, "operator": "NotIn",
                                 "values": [unique_key]}]},
    }
