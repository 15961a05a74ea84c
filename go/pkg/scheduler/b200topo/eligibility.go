/*
Copyright 2024 The RoleBasedGroup Authors.

Licensed under the Apache License, Version 2.0 (the "License").
*/

package b200topo

// Node eligibility (DESIGN.md §3.19): nodes grouped into classes whose configured label values and NoSchedule /
// NoExecute taints are equal, and one class mask per role from its pod template.  The mirror of
// rbg_b200/ingest.py::build_node_classes / role_admit; the selector rules are upstream's own (nodeaffinity, the
// Toleration method), evaluated against one representative node per class.

import (
	"fmt"
	"sort"

	corev1 "k8s.io/api/core/v1"
	"k8s.io/component-helpers/scheduling/corev1/nodeaffinity"
	workloadsv1alpha2 "sigs.k8s.io/rbgs/api/workloads/v1alpha2"
)

// maxNodeClasses = RBGTOPO_MAX_NODE_CLASSES.
const maxNodeClasses = 64

type nodeClasses struct {
	keys   []string
	class  []int32             // per node id
	labels []map[string]string // per class: the configured keys' values
	taints [][]corev1.Taint    // per class: its NoSchedule / NoExecute taints
}

func hardTaints(ts []corev1.Taint) []corev1.Taint {
	var out []corev1.Taint
	for _, t := range ts {
		if t.Effect == corev1.TaintEffectNoSchedule || t.Effect == corev1.TaintEffectNoExecute {
			out = append(out, corev1.Taint{Key: t.Key, Value: t.Value, Effect: t.Effect})
		}
	}
	sort.Slice(out, func(a, b int) bool {
		x, y := out[a], out[b]
		if x.Key != y.Key {
			return x.Key < y.Key
		}
		if x.Value != y.Value {
			return x.Value < y.Value
		}
		return x.Effect < y.Effect
	})
	return out
}

// buildNodeClasses numbers classes by first appearance over the snapshot's name-sorted nodes, so the result does not
// depend on informer order; more than maxNodeClasses is an error (configure fewer keys).
func buildNodeClasses(names []string, nodes map[string]*nodeInfo, keys []string) (*nodeClasses, error) {
	c := &nodeClasses{keys: keys, class: make([]int32, len(names))}
	ids := map[string]int32{}
	for i, nm := range names {
		ni := nodes[nm]
		lab := map[string]string{}
		sig := ""
		for _, k := range keys {
			if v, ok := ni.labels[k]; ok {
				lab[k] = v
				sig += fmt.Sprintf("%q=%q;", k, v)
			} else {
				sig += fmt.Sprintf("%q!;", k)
			}
		}
		ts := hardTaints(ni.taints)
		for _, t := range ts {
			sig += fmt.Sprintf("|%q=%q:%s", t.Key, t.Value, t.Effect)
		}
		id, ok := ids[sig]
		if !ok {
			id = int32(len(c.labels))
			ids[sig] = id
			c.labels = append(c.labels, lab)
			c.taints = append(c.taints, ts)
		}
		c.class[i] = id
	}
	if len(c.labels) > maxNodeClasses {
		return nil, fmt.Errorf("%d node classes exceed %d: configure fewer label keys", len(c.labels), maxNodeClasses)
	}
	return c, nil
}

// roleAdmit: bit c set when class c admits the template (nodeSelector, required node affinity, hard taints), or a
// reason when a selector key is outside the configured keys or a term uses matchFields.
func (c *nodeClasses) roleAdmit(spec *corev1.PodSpec) (uint64, string) {
	known := map[string]bool{}
	for _, k := range c.keys {
		known[k] = true
	}
	for k := range spec.NodeSelector {
		if !known[k] {
			return 0, "node eligibility: nodeSelector key " + k + " is not a configured class key"
		}
	}
	if a := spec.Affinity; a != nil && a.NodeAffinity != nil && a.NodeAffinity.RequiredDuringSchedulingIgnoredDuringExecution != nil {
		for _, term := range a.NodeAffinity.RequiredDuringSchedulingIgnoredDuringExecution.NodeSelectorTerms {
			if len(term.MatchFields) > 0 {
				return 0, "node eligibility: node affinity matchFields cannot be decided per class"
			}
			for _, e := range term.MatchExpressions {
				if !known[e.Key] {
					return 0, "node eligibility: node affinity key " + e.Key + " is not a configured class key"
				}
			}
		}
	}
	pod := &corev1.Pod{Spec: *spec}
	req := nodeaffinity.GetRequiredNodeAffinity(pod)
	var mask uint64
	for cl := range c.labels {
		node := &corev1.Node{}
		node.Labels = c.labels[cl]
		if ok, err := req.Match(node); err != nil || !ok {
			continue
		}
		tolerated := true
		for i := range c.taints[cl] {
			t := &c.taints[cl][i]
			one := false
			for j := range spec.Tolerations {
				if spec.Tolerations[j].ToleratesTaint(t) {
					one = true
					break
				}
			}
			if !one {
				tolerated = false
				break
			}
		}
		if tolerated {
			mask |= 1 << uint(cl)
		}
	}
	return mask, ""
}

// roleMasks: the mask of every role in rbg.Spec.Roles order, whether one excludes an installed class, or a reason.
func (c *nodeClasses) roleMasks(rbg *workloadsv1alpha2.RoleBasedGroup) ([]uint64, bool, string) {
	full := uint64(1)<<uint(len(c.labels)) - 1
	if len(c.labels) == 64 {
		full = ^uint64(0)
	}
	out := make([]uint64, len(rbg.Spec.Roles))
	restricted := false
	for i := range rbg.Spec.Roles {
		spec := &corev1.PodSpec{}
		if t := rbg.Spec.Roles[i].GetTemplate(); t != nil {
			spec = &t.Spec
		}
		m, reason := c.roleAdmit(spec)
		if reason != "" {
			return nil, false, reason
		}
		out[i] = m
		restricted = restricted || m&full != full
	}
	return out, restricted, ""
}

// SetNodeClassKeys turns node eligibility on (DESIGN.md §3.19): nodes are grouped by the values of these label keys
// and their hard taints, the classes are installed after every topology upload, and a group with a role whose pod
// template excludes a class is placed through rbgtopo_place_groups_eligible[_ranked].  nil (the default) turns it off.
func (m *Manager) SetNodeClassKeys(keys []string) {
	m.nodes.mu.Lock()
	defer m.nodes.mu.Unlock()
	m.nodes.classKeys = append([]string(nil), keys...) // nil stays nil
	m.nodes.topoGen++ // the next sync uploads the topology and its classes
}
