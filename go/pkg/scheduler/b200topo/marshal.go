/*
Copyright 2024 The RoleBasedGroup Authors.

Licensed under the Apache License, Version 2.0 (the "License").
*/

package b200topo

import (
	"fmt"
	"sort"

	corev1 "k8s.io/api/core/v1"
	"sigs.k8s.io/rbgs/api/workloads/constants"
	workloadsv1alpha2 "sigs.k8s.io/rbgs/api/workloads/v1alpha2"
)

// GROUPS wire format of include/rbgtopo.h.
const (
	groupsMagic   = 0x47474252
	abiVersion    = 1
	hdrWords      = 8
	groupWords    = 12
	stepExclusive = 1
	stepGang      = 2
	roleExclusive = 1
	maxGroupRoles = 16
)

// DemandResource is the accelerator resource whose request is a replica's `demand`.
const DemandResource = corev1.ResourceName("nvidia.com/gpu")

type marshalled struct {
	blob    []int32
	pending int
	order   []int    // role indices sorted by (level, name): the blob's role order
	first   []int32  // first pending ordinal per role (= replicas that exist already)
	count   []int32  // pending replicas per role
	names   []string // role names, rbg.Spec.Roles order
	rbgName string
}

// dependencyLevels restates dependencyOrder (pkg/dependency/dependency.go:129-205, unexported):
// names sorted first, level = 1 + max(level of the dependencies), cycle => error.  Pinned to the
// reference's own table test by the C mirror rbgtopo_dependency_levels (tests/test_host_pinned.py).
func dependencyLevels(deps map[string][]string) (map[string]int, error) {
	names := make([]string, 0, len(deps))
	for n := range deps {
		names = append(names, n)
	}
	sort.Strings(names)
	level := map[string]int{}
	state := map[string]int{} // 1 = on the stack, 2 = done
	var visit func(string) (int, error)
	visit = func(n string) (int, error) {
		switch state[n] {
		case 2:
			return level[n], nil
		case 1:
			return 0, fmt.Errorf("cycle detected for role '%s'", n)
		}
		state[n] = 1
		mx := 0
		for _, d := range deps[n] {
			if _, ok := deps[d]; !ok {
				return 0, fmt.Errorf("dependency '%s' not found for role '%s'", d, n)
			}
			l, err := visit(d)
			if err != nil {
				return 0, err
			}
			if l+1 > mx {
				mx = l + 1
			}
		}
		state[n], level[n] = 2, mx
		return mx, nil
	}
	for _, n := range names {
		if _, err := visit(n); err != nil {
			return nil, err
		}
	}
	return level, nil
}

// marshalGroup builds the one-group GROUPS blob of rbg (INTEGRATION.md §3 lists the source of every
// field).  targets: coordination scaling targets when a CoordinatedPolicy paces the group
// (CalculateScalingForAllCoordination, rolebasedgroup_controller.go:968-1054), else spec replicas.
func marshalGroup(rbg *workloadsv1alpha2.RoleBasedGroup, pods []corev1.Pod, snap *snapshot, gid int32) (*marshalled, error) {
	roles := rbg.Spec.Roles
	q := len(roles)
	if q == 0 || q > maxGroupRoles {
		return nil, fmt.Errorf("b200topo: %d roles (limit %d)", q, maxGroupRoles)
	}
	deps := map[string][]string{}
	index := map[string]int{}
	for i := range roles {
		deps[roles[i].Name] = roles[i].Dependencies
		index[roles[i].Name] = i
	}
	levels, err := dependencyLevels(deps)
	if err != nil {
		return nil, err
	}
	order := make([]int, q)
	for i := range order {
		order[i] = i
	}
	sort.Slice(order, func(a, b int) bool {
		la, lb := levels[roles[order[a]].Name], levels[roles[order[b]].Name]
		if la != lb {
			return la < lb
		}
		return roles[order[a]].Name < roles[order[b]].Name
	})
	pos := make([]int, q) // role index -> position in the blob
	for k, ri := range order {
		pos[ri] = k
	}
	m := &marshalled{order: order, first: make([]int32, q), count: make([]int32, q), names: make([]string, q), rbgName: rbg.Name}
	// pair matrix (DESIGN.md §3.2): same role, dependency edge, both in one CoordinatedPolicy rule
	pair := make([]int32, q*q)
	for i := range roles {
		pair[pos[i]*q+pos[i]] = 1
		for _, d := range roles[i].Dependencies {
			pair[pos[i]*q+pos[index[d]]], pair[pos[index[d]]*q+pos[i]] = 1, 1
		}
	}
	for _, rule := range coordinatedRoleSets(rbg) {
		for _, a := range rule {
			for _, b := range rule {
				ia, oka := index[a]
				ib, okb := index[b]
				if oka && okb {
					pair[pos[ia]*q+pos[ib]] = 1
				}
			}
		}
	}
	flags := int32(0)
	if _, ok := rbg.GetExclusiveKey(); ok { // annotation.go:25
		flags |= stepExclusive
	}
	if rbg.Annotations[constants.GangSchedulingAnnotationKey] == "true" { // annotation.go:37
		flags |= stepGang
	}
	roleRecs := make([]int32, 0, 4*q)
	for _, ri := range order {
		role := &roles[ri]
		m.names[ri] = role.Name
		cur := int32(0)
		if st, ok := rbg.GetRoleStatus(role.Name); ok {
			cur = st.Replicas
		}
		tgt := int32(1)
		if role.Replicas != nil {
			tgt = *role.Replicas
		}
		pend := tgt - cur
		if pend < 0 {
			pend = 0
		}
		m.first[ri], m.count[ri] = cur, pend
		m.pending += int(pend)
		rf := int32(roleExclusive)
		if role.Annotations[constants.RoleDisableExclusiveKey] == "true" { // annotation.go:29, pod_reconciler.go:127
			rf = 0
		}
		roleRecs = append(roleRecs, int32(levels[role.Name]), pend, demandOf(role), rf)
	}
	// anchors: scheduled pods of the group (node, role position, 1); fixed domain = domain of any of them
	var anchors []int32
	fixed := int32(-1)
	for i := range pods {
		roleName := pods[i].Labels[constants.RoleNameLabelKey]
		ri, ok := index[roleName]
		node, okn := snap.nodeID(pods[i].Spec.NodeName)
		if !ok || !okn {
			continue
		}
		anchors = append(anchors, node, int32(pos[ri]), 1)
		if flags&stepExclusive != 0 && fixed < 0 {
			fixed = snap.domain[node]
		}
	}
	base := hdrWords + groupWords
	roleOff := base
	pairOff := roleOff + len(roleRecs)
	anchorOff := pairOff + len(pair)
	words := anchorOff + len(anchors)
	blob := make([]int32, 0, words)
	blob = append(blob, groupsMagic, abiVersion, 1, int32(words), int32(m.pending), 0, 0, 0)
	blob = append(blob, gid, flags, fixed, int32(q), int32(roleOff), int32(pairOff), int32(len(anchors)/3), int32(anchorOff),
		0, int32(m.pending), 0, 0) // +10 exclusive level 0: Manager.exclusiveLevel keeps other keys out
	blob = append(blob, roleRecs...)
	blob = append(blob, pair...)
	blob = append(blob, anchors...)
	m.blob = blob
	return m, nil
}

// roleIDMap: assign[] is in (blob role order, ordinal) order; RoleID "{rbg}-{role}-{ordinal}"
// (api/workloads/v1alpha2/helper.go:68-81, stateful_instance_set_utils.go:74-76).  A gang failure
// (status 2) yields an empty map: all-or-nothing (k8s-scheduler-plugin/manager.go:131).
func (m *marshalled) roleIDMap(assign []int32, snap *snapshot, status int32) map[string]string {
	out := map[string]string{}
	if status == 2 {
		return out
	}
	k := 0
	for _, ri := range m.order {
		for c := int32(0); c < m.count[ri]; c++ {
			if node := assign[k]; node >= 0 {
				out[fmt.Sprintf("%s-%s-%d", m.rbgName, m.names[ri], m.first[ri]+c)] = snap.names[node]
			}
			k++
		}
	}
	return out
}

// roleIDAlternates: altNode[] holds nAlt node indices per replica in assign order (-1 = none); RoleID -> node names,
// replicas without alternates left out.  A gang failure yields an empty map, like roleIDMap.
func (m *marshalled) roleIDAlternates(altNode []int32, nAlt int, snap *snapshot, status int32) map[string][]string {
	out := map[string][]string{}
	if status == 2 {
		return out
	}
	k := 0
	for _, ri := range m.order {
		for c := int32(0); c < m.count[ri]; c++ {
			var names []string
			for _, node := range altNode[k*nAlt : (k+1)*nAlt] {
				if node >= 0 {
					names = append(names, snap.names[node])
				}
			}
			if len(names) > 0 {
				out[fmt.Sprintf("%s-%s-%d", m.rbgName, m.names[ri], m.first[ri]+c)] = names
			}
			k++
		}
	}
	return out
}

func demandOf(role *workloadsv1alpha2.RoleSpec) int32 {
	t := role.GetTemplate()
	if t == nil {
		return 0
	}
	var d int64
	for i := range t.Spec.Containers {
		if v, ok := t.Spec.Containers[i].Resources.Requests[DemandResource]; ok {
			d += v.Value()
		}
	}
	if d > 32767 {
		d = 32767 // RBGTOPO_MAX_FREE
	}
	return int32(d)
}

// coordinatedRoleSets: the role sets of the CoordinatedPolicy rules that pace this group
// (api/workloads/v1alpha2/coordinatedpolicy_types.go:41-45).  The controller already holds the
// policy at step 5 of Reconcile; the manager receives it through the RBG's annotations cache in the
// full patch — here the hook is a function variable so that the file stands alone.
var coordinatedRoleSets = func(rbg *workloadsv1alpha2.RoleBasedGroup) [][]string { return nil }
