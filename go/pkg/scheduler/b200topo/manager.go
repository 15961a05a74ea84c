/*
Copyright 2024 The RoleBasedGroup Authors.

Licensed under the Apache License, Version 2.0 (the "License").
*/

// Package b200topo is a third implementation of scheduler.PodGroupManager
// (pkg/scheduler/podgroup_manager.go:64-78): it keeps the PodGroup CR bookkeeping of the wrapped
// kube / volcano implementation and additionally computes topology-aware placement hints for the
// group's pending replicas on an H100 through librbgtopo.so (include/rbgtopo.h).
//
// Wiring (the only edits to reference code, INTEGRATION.md §1):
//
//	const B200TopoPlugin SchedulerPluginType = "b200-topo"
//	case B200TopoPlugin: return b200topo.New(c, kubeschedulerplugin.New(c)), nil
//
// NOT COMPILED IN THE BUILD IMAGE OF THIS REPO (no Go toolchain): source for a maintainer; the
// same logic runs in rbg_b200/plugin.py over ctypes and is what the tests exercise.
package b200topo

import (
	"context"
	"encoding/json"
	"sync"

	corev1 "k8s.io/api/core/v1"
	coreapplyv1 "k8s.io/client-go/applyconfigurations/core/v1"
	"sigs.k8s.io/controller-runtime/pkg/builder"
	"sigs.k8s.io/controller-runtime/pkg/client"
	"sigs.k8s.io/controller-runtime/pkg/log"
	"sigs.k8s.io/controller-runtime/pkg/reconcile"
	workloadsv1alpha2 "sigs.k8s.io/rbgs/api/workloads/v1alpha2"
)

// PlacementHintKey carries the serialized RoleID -> node-name map on the pod template
// (InjectPodGroupLabels sees a template, not a replica: SURVEY.md §8b "Injection into L4").
const PlacementHintKey = "rbg.workloads.x-k8s.io/b200-topo-placement"

// PlacementAlternatesKey carries RoleID -> ranked next-best node names (DESIGN.md §3.10) beside the hint, written only
// when the manager is configured with alternates (SetAlternates) and only for replicas that have some.
const PlacementAlternatesKey = "rbg.workloads.x-k8s.io/b200-topo-alternates"

// inner is the part of scheduler.PodGroupManager this package wraps (declared here to avoid an
// import cycle with pkg/scheduler, which imports this package in its factory).
type inner interface {
	ReconcilePodGroup(ctx context.Context, rbg *workloadsv1alpha2.RoleBasedGroup,
		runtimeController *builder.TypedBuilder[reconcile.Request], watchedWorkload *sync.Map, apiReader client.Reader) error
	InjectPodGroupLabels(rbg *workloadsv1alpha2.RoleBasedGroup, pts *coreapplyv1.PodTemplateSpecApplyConfiguration)
}

// Manager implements scheduler.PodGroupManager.
type Manager struct {
	client client.Client
	inner  inner      // kube or volcano implementation: still owns the PodGroup CR
	placer *placer    // nil => degraded: behaves exactly like `inner`
	nodes  *nodeCache // Node informer -> CSR + free / domain arrays (nodecache.go)
	hints  sync.Map   // "ns/name" -> map[RoleID]string (node name)
	gids   gidTable   // dense group ids (domain_owner[] compares against them)
	// exclusiveKeys: the topology keys exclusive groups may name (DESIGN.md §3.9), keys[0] = the level-0 label.
	// nil: every key is treated as the level-0 label (the behaviour before levels existed).
	exclusiveKeys []string
	// alternates: next-best nodes per replica carried beside the hint (0 = the single-node hint of before, at most
	// RBGTOPO_MAX_ALTERNATES); alts holds them per group like hints
	alternates int
	alts       sync.Map // "ns/name" -> map[RoleID][]string (node names)
}

// SetAlternates configures how many ranked next-best nodes every hinted replica carries (DESIGN.md §3.10): 0 (the
// default) keeps the single-node hint and the call made; n in [1, 8] places through rbgtopo_place_groups_ranked, which
// places identically.  Values outside [0, 8] are clamped.
func (m *Manager) SetAlternates(n int) { m.alternates = min(max(n, 0), 8) }

// SetExclusiveKeys configures the topology keys exclusive groups may name; keys[0] must be the level-0 label (the
// first tier label of the node cache).  nil restores the behaviour without levels.
func (m *Manager) SetExclusiveKeys(keys []string) { m.exclusiveKeys = append([]string(nil), keys...) }

// exclusiveLevel: the level of an exclusive group's key, or a reason for giving it no hint.  The library places
// level-0 groups only, and a hint into a domain of the wrong key is worse than none (kube-scheduler enforces the
// group's required terms on its own key).
func (m *Manager) exclusiveLevel(rbg *workloadsv1alpha2.RoleBasedGroup) (int32, string) {
	key, ok := rbg.GetExclusiveKey()
	if !ok || m.exclusiveKeys == nil {
		return 0, ""
	}
	for i, k := range m.exclusiveKeys {
		if k == key {
			if i == 0 {
				return 0, ""
			}
			return int32(i), "exclusive key " + key + " is not the level-0 label: no placement at that level yet"
		}
	}
	return -1, "exclusive key " + key + " is not configured"
}

// New never fails: without an H100 (RBGTOPO_ENODEVICE) or without the library the manager degrades
// to the wrapped implementation — the controller's behaviour today.
func New(c client.Client, in inner) *Manager {
	m := &Manager{client: c, inner: in, nodes: newNodeCache()}
	p, err := newPlacer(0)
	if err != nil {
		log.Log.WithName("b200topo").Info("no placement hints: " + err.Error())
		return m
	}
	m.placer = p
	return m
}

// ReconcilePodGroup — step 6 of Reconcile (rolebasedgroup_controller.go:200-204, :422-430).
func (m *Manager) ReconcilePodGroup(ctx context.Context, rbg *workloadsv1alpha2.RoleBasedGroup,
	runtimeController *builder.TypedBuilder[reconcile.Request], watchedWorkload *sync.Map, apiReader client.Reader) error {
	if err := m.inner.ReconcilePodGroup(ctx, rbg, runtimeController, watchedWorkload, apiReader); err != nil {
		return err
	}
	if m.placer == nil {
		return nil
	}
	logger := log.FromContext(ctx).WithName("b200topo")
	key := rbg.Namespace + "/" + rbg.Name
	snap, err := m.nodes.sync(m.placer) // set_topology / update_nodes[_delta], keyed by generation
	if err != nil {
		return m.degrade(logger, key, err)
	}
	pods, err := m.scheduledPods(ctx, rbg)
	if err != nil {
		return err // an API error: requeue like every other LIST failure of the controller
	}
	if _, reason := m.exclusiveLevel(rbg); reason != "" {
		m.hints.Delete(key)
		m.alts.Delete(key)
		logger.Info("no placement hint", "rbg", key, "reason", reason)
		return nil
	}
	g, err := marshalGroup(rbg, pods, snap, m.gids.id(rbg))
	if err != nil {
		return err // cycle in the role dependencies etc.: the controller reports the same condition
	}
	if g.pending == 0 {
		return nil
	}
	if m.alternates > 0 {
		assign, status, _, altNode, err := m.placer.placeGroupsRanked(g.blob, m.alternates)
		if err != nil {
			return m.degrade(logger, key, err)
		}
		m.hints.Store(key, g.roleIDMap(assign, snap, status[0]))
		m.alts.Store(key, g.roleIDAlternates(altNode, m.alternates, snap, status[0]))
		return nil
	}
	assign, status, _, err := m.placer.placeGroups(g.blob)
	if err != nil {
		return m.degrade(logger, key, err)
	}
	m.hints.Store(key, g.roleIDMap(assign, snap, status[0]))
	return nil
}

// degrade: device trouble (RBGTOPO_ECUDA / _ENODEVICE) must never block the reconcile — drop the
// hint and carry on (SURVEY.md §8b: "a CUDA failure must degrade to no placement"); malformed
// input is the shim's own bug or a spec limit: log it, no hint, no requeue loop either.
func (m *Manager) degrade(logger interface{ Info(string, ...any) }, key string, err error) error {
	m.hints.Delete(key)
	m.alts.Delete(key)
	if pe, ok := err.(*placerError); ok && pe.deviceTrouble() {
		logger.Info("placement hints disabled for this reconcile", "rbg", key, "reason", pe.Error())
		return nil
	}
	logger.Info("no placement hint", "rbg", key, "reason", err.Error())
	return nil
}

// InjectPodGroupLabels — pkg/reconciler/pod_reconciler.go:150-153.
func (m *Manager) InjectPodGroupLabels(rbg *workloadsv1alpha2.RoleBasedGroup, pts *coreapplyv1.PodTemplateSpecApplyConfiguration) {
	m.inner.InjectPodGroupLabels(rbg, pts)
	if h, ok := m.hints.Load(rbg.Namespace + "/" + rbg.Name); ok {
		if b, err := json.Marshal(h); err == nil {
			pts.WithAnnotations(map[string]string{PlacementHintKey: string(b)})
		}
	}
	if a, ok := m.alts.Load(rbg.Namespace + "/" + rbg.Name); ok && len(a.(map[string][]string)) > 0 {
		if b, err := json.Marshal(a); err == nil {
			pts.WithAnnotations(map[string]string{PlacementAlternatesKey: string(b)})
		}
	}
}

// NodeHintFor is the per-replica half of the write-back (SURVEY.md §8f rank 2): the hook in
// createPods (pkg/reconciler/roleinstance/sync/instance_scale.go:129-186, see hints.go) asks for the
// node of ONE pod; the template annotation above is only the fallback every replica shares.
func (m *Manager) NodeHintFor(namespace, rbgName, roleID string) (string, bool) {
	h, ok := m.hints.Load(namespace + "/" + rbgName)
	if !ok {
		return "", false
	}
	node, ok := h.(map[string]string)[roleID]
	return node, ok
}

// scheduledPods: the LIST of getScheduledReplicas (rolebasedgroup_controller.go:1057-1080), kept.
func (m *Manager) scheduledPods(ctx context.Context, rbg *workloadsv1alpha2.RoleBasedGroup) ([]corev1.Pod, error) {
	var out []corev1.Pod
	for i := range rbg.Spec.Roles {
		role := &rbg.Spec.Roles[i]
		var pods corev1.PodList
		if err := m.client.List(ctx, &pods, client.InNamespace(rbg.Namespace),
			client.MatchingLabels(rbg.GetCommonLabelsFromRole(role))); err != nil {
			return nil, err
		}
		for j := range pods.Items {
			if pods.Items[j].Spec.NodeName != "" && pods.Items[j].DeletionTimestamp == nil {
				out = append(out, pods.Items[j])
			}
		}
	}
	return out, nil
}

// gidTable hands out dense group ids; GenGroupUniqueKey (api/workloads/v1alpha2/helper.go:135-144)
// is the stable key.
type gidTable struct {
	mu   sync.Mutex
	ids  map[string]int32
	next int32
}

func (t *gidTable) id(rbg *workloadsv1alpha2.RoleBasedGroup) int32 {
	t.mu.Lock()
	defer t.mu.Unlock()
	if t.ids == nil {
		t.ids = map[string]int32{}
	}
	k := rbg.GenGroupUniqueKey()
	if v, ok := t.ids[k]; ok {
		return v
	}
	t.ids[k] = t.next
	t.next++
	return t.ids[k]
}
