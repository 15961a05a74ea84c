/*
Copyright 2024 The RoleBasedGroup Authors.

Licensed under the Apache License, Version 2.0 (the "License").
*/

package b200topo

import (
	"encoding/json"

	corev1 "k8s.io/api/core/v1"
)

// Per-replica hint write-back (SURVEY.md §8f rank 2).  InjectPodGroupLabels sees a pod TEMPLATE, so
// the annotation it writes carries the whole RoleID -> node map and every replica shares it.  The
// replica-specific half happens where pods are created, in createPods
// (pkg/reconciler/roleinstance/sync/instance_scale.go:129-186), right after the port injection
// (:164-169):
//
//	// + b200-topo: turn the group's placement map into a preference of THIS pod
//	b200topo.ApplyNodeHint(p)
//
// ApplyNodeHint reads the map from the pod's own annotations (inherited from the template), looks
// up the pod's RoleID — its name, "{rbg}-{role}-{ordinal}" for standalone instances
// (pkg/reconciler/roleinstance/utils/instance_utils.go:76-89) — and adds a PREFERRED node-affinity
// term on kubernetes.io/hostname.  Preferred, not required: kube-scheduler / the gang plugin still
// bind the pod and arbitrate conflicts between concurrent reconciles (DESIGN.md §3.7).
//
// With the alternates annotation (Manager.SetAlternates, DESIGN.md §3.10) the pod also gets one preferred term per
// ranked next-best node, alternate i of F listed for the pod with weight max(1, 100*(F-i)/(F+1)): below the primary's
// 100 and descending, so a pod whose hinted node filled up before it was bound still lands on the next-best node of
// its own row that had room once its group was placed.
const hintWeight = 100

func ApplyNodeHint(p *corev1.Pod) bool {
	raw, ok := p.Annotations[PlacementHintKey]
	if !ok {
		return false
	}
	var m map[string]string
	if err := json.Unmarshal([]byte(raw), &m); err != nil {
		return false
	}
	node, ok := m[p.Name]
	if !ok || node == "" {
		return false
	}
	term := corev1.PreferredSchedulingTerm{
		Weight: hintWeight,
		Preference: corev1.NodeSelectorTerm{MatchExpressions: []corev1.NodeSelectorRequirement{{
			Key: corev1.LabelHostname, Operator: corev1.NodeSelectorOpIn, Values: []string{node},
		}}},
	}
	if p.Spec.Affinity == nil {
		p.Spec.Affinity = &corev1.Affinity{}
	}
	if p.Spec.Affinity.NodeAffinity == nil {
		p.Spec.Affinity.NodeAffinity = &corev1.NodeAffinity{}
	}
	na := p.Spec.Affinity.NodeAffinity
	na.PreferredDuringSchedulingIgnoredDuringExecution = append(na.PreferredDuringSchedulingIgnoredDuringExecution, term)
	delete(p.Annotations, PlacementHintKey) // the map of the whole group does not need to live on every pod
	if raw, ok := p.Annotations[PlacementAlternatesKey]; ok {
		var alts map[string][]string
		if err := json.Unmarshal([]byte(raw), &alts); err == nil {
			nodes := alts[p.Name]
			f := int32(len(nodes))
			for i, n := range nodes {
				na.PreferredDuringSchedulingIgnoredDuringExecution = append(na.PreferredDuringSchedulingIgnoredDuringExecution,
					corev1.PreferredSchedulingTerm{
						Weight: max(1, hintWeight*(f-int32(i))/(f+1)),
						Preference: corev1.NodeSelectorTerm{MatchExpressions: []corev1.NodeSelectorRequirement{{
							Key: corev1.LabelHostname, Operator: corev1.NodeSelectorOpIn, Values: []string{n},
						}}},
					})
			}
		}
		delete(p.Annotations, PlacementAlternatesKey)
	}
	return true
}
