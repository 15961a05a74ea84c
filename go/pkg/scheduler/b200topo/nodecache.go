/*
Copyright 2024 The RoleBasedGroup Authors.

Licensed under the Apache License, Version 2.0 (the "License").
*/

package b200topo

import (
	"sort"
	"sync"

	corev1 "k8s.io/api/core/v1"
	toolscache "k8s.io/client-go/tools/cache"
)

// Node-topology ingestion (SURVEY.md §8f rank 1).  The reference has no Node informer
// (the controller never lists Nodes; RBAC markers rolebasedgroup_controller.go:103-127 name no
// `nodes`), so this file is new:
//
//	// +kubebuilder:rbac:groups="",resources=nodes,verbs=get;list;watch
//
// and, next to the cache options of cmd/rbgs/main.go:408-429, the manager is started with
//
//	nodeInformer, _ := mgr.GetCache().GetInformer(ctx, &corev1.Node{})
//	podInformer, _  := mgr.GetCache().GetInformer(ctx, &corev1.Pod{})
//	pgm.(*b200topo.Manager).RegisterInformers(nodeInformer, podInformer)
//
// rbg_b200/ingest.py is this file rule for rule (tests/test_ingest.py pins the rules:
// determinism under informer reordering, symmetric sorted CSR, closest tier wins).
//
// Label conventions (closest tier first).  The first one is also the exclusive-topology domain
// (rbg.workloads.x-k8s.io/group-exclusive-topology names a topology key, annotation.go:25).
var TierLabels = []string{
	"nvidia.com/nvlink-domain",     // NVL72 / NVSwitch domain
	"kubernetes.io/hostname-group", // hosts behind one PCIe / NIC complex
	"network.topology/rdma-leaf",   // RDMA leaf switch
	"topology.kubernetes.io/zone",  // VPC / zone
}

// TierWeights: NVLink > PCIe > RDMA > VPC (README.md:53 order; magnitudes: DESIGN.md §3.1).
var TierWeights = []int32{1000, 100, 10, 1}

// TierFanout: links per node and tier (the whole NVL72 domain; name-order successors above).
var TierFanout = []int{71, 8, 8, 4}

const maxFree = 32767 // RBGTOPO_MAX_FREE

type nodeInfo struct {
	labels        map[string]string
	allocatable   int64
	requested     int64 // summed over the node's non-terminated pods
	unschedulable bool
	taints        []corev1.Taint // spec.taints (node eligibility, eligibility.go)
}

// snapshot = the arrays of rbgtopo_set_topology, immutable once built.
type snapshot struct {
	names                                      []string // id -> node name
	ids                                        map[string]int32
	domains                                    []string
	rowPtr, colIdx, edgeW, free, domain, owner []int32
	topoGen, capGen                            uint64
	classes                                    *nodeClasses // nil: node eligibility off (Manager.SetNodeClassKeys)
}

func (s *snapshot) nodeID(name string) (int32, bool) { id, ok := s.ids[name]; return id, ok }

type nodeCache struct {
	mu                    sync.Mutex
	nodes                 map[string]*nodeInfo
	domainOwner           map[string]int32 // domain name -> gid of the group holding it exclusively
	topoGen, capGen       uint64           // bumped by the informer handlers
	pushedTopo, pushedCap uint64
	snap                  *snapshot
	dirty                 map[string]struct{} // nodes whose capacity changed since the last push
	classKeys             []string            // node eligibility: the label keys of the node classes (nil: off)
}

func newNodeCache() *nodeCache {
	return &nodeCache{nodes: map[string]*nodeInfo{}, domainOwner: map[string]int32{}, dirty: map[string]struct{}{}}
}

// RegisterInformers wires the handlers; event order does not matter (ids by name, groups by label value).
func (m *Manager) RegisterInformers(nodeInformer, podInformer toolscache.SharedIndexInformer) {
	nc := m.nodes
	_, _ = nodeInformer.AddEventHandler(toolscache.ResourceEventHandlerFuncs{
		AddFunc:    func(o any) { nc.upsertNode(o.(*corev1.Node)) },
		UpdateFunc: func(_, o any) { nc.upsertNode(o.(*corev1.Node)) },
		DeleteFunc: func(o any) {
			if n, ok := o.(*corev1.Node); ok {
				nc.deleteNode(n.Name)
			}
		},
	})
	_, _ = podInformer.AddEventHandler(toolscache.ResourceEventHandlerFuncs{
		AddFunc:    func(o any) { nc.podDelta(o.(*corev1.Pod), +1) },
		DeleteFunc: func(o any) {
			if p, ok := o.(*corev1.Pod); ok {
				nc.podDelta(p, -1)
			}
		},
	})
}

func tierKeyChanged(a, b map[string]string) bool {
	for _, k := range TierLabels {
		if a[k] != b[k] {
			return true
		}
	}
	return false
}

func (nc *nodeCache) upsertNode(n *corev1.Node) {
	nc.mu.Lock()
	defer nc.mu.Unlock()
	alloc := n.Status.Allocatable[DemandResource]
	ready := false
	for _, c := range n.Status.Conditions {
		if c.Type == corev1.NodeReady && c.Status == corev1.ConditionTrue {
			ready = true
		}
	}
	old, ok := nc.nodes[n.Name]
	ni := &nodeInfo{labels: n.Labels, allocatable: alloc.Value(), unschedulable: n.Spec.Unschedulable || !ready,
		taints: n.Spec.Taints}
	if ok {
		ni.requested = old.requested
	}
	nc.nodes[n.Name] = ni
	switch {
	case !ok || tierKeyChanged(old.labels, ni.labels) || nc.classChanged(old, ni):
		nc.topoGen++ // node SET or a tier label changed: the CSR is rebuilt (rbgtopo_set_topology)
	case old.allocatable != ni.allocatable || old.unschedulable != ni.unschedulable:
		nc.capGen++ // capacity churn only (rbgtopo_update_nodes[_delta])
		nc.dirty[n.Name] = struct{}{}
	}
}

func (nc *nodeCache) deleteNode(name string) {
	nc.mu.Lock()
	defer nc.mu.Unlock()
	if _, ok := nc.nodes[name]; ok {
		delete(nc.nodes, name)
		nc.topoGen++
	}
}

func (nc *nodeCache) podDelta(p *corev1.Pod, sign int64) {
	if p.Spec.NodeName == "" {
		return
	}
	var req int64
	for i := range p.Spec.Containers {
		if v, ok := p.Spec.Containers[i].Resources.Requests[DemandResource]; ok {
			req += v.Value()
		}
	}
	if req == 0 {
		return
	}
	nc.mu.Lock()
	defer nc.mu.Unlock()
	if ni, ok := nc.nodes[p.Spec.NodeName]; ok {
		ni.requested += sign * req
		nc.capGen++
		nc.dirty[p.Spec.NodeName] = struct{}{}
	}
}

func freeSlots(ni *nodeInfo) int32 {
	if ni.unschedulable {
		return 0
	}
	f := ni.allocatable - ni.requested
	if f < 0 {
		f = 0
	}
	if f > maxFree {
		f = maxFree
	}
	return int32(f)
}

type edge struct {
	a, b, w int32
}

// build: rbg_b200/ingest.py::build_topology.
func (nc *nodeCache) build() *snapshot {
	names := make([]string, 0, len(nc.nodes))
	for n := range nc.nodes {
		names = append(names, n)
	}
	sort.Strings(names)
	s := &snapshot{names: names, ids: make(map[string]int32, len(names)), topoGen: nc.topoGen, capGen: nc.capGen}
	for i, n := range names {
		s.ids[n] = int32(i)
	}
	var edges []edge
	for tier, key := range TierLabels {
		groups := map[string][]int32{}
		for i, n := range names { // ascending ids = name order
			if v, ok := nc.nodes[n].labels[key]; ok {
				groups[v] = append(groups[v], int32(i))
			}
		}
		for _, mem := range groups {
			m := len(mem)
			if m < 2 {
				continue
			}
			k := TierFanout[tier]
			if k > m-1 {
				k = m - 1
			}
			for off := 1; off <= k; off++ {
				for i := range mem {
					a, b := mem[i], mem[(i+off)%m]
					if a != b {
						edges = append(edges, edge{a, b, TierWeights[tier]}, edge{b, a, TierWeights[tier]})
					}
				}
			}
		}
	}
	// a pair keeps its closest tier = largest weight
	sort.Slice(edges, func(i, j int) bool {
		if edges[i].a != edges[j].a {
			return edges[i].a < edges[j].a
		}
		if edges[i].b != edges[j].b {
			return edges[i].b < edges[j].b
		}
		return edges[i].w > edges[j].w
	})
	n := len(names)
	s.rowPtr = make([]int32, n+1)
	for i, e := range edges {
		if i > 0 && edges[i-1].a == e.a && edges[i-1].b == e.b {
			continue
		}
		s.colIdx = append(s.colIdx, e.b)
		s.edgeW = append(s.edgeW, e.w)
		s.rowPtr[e.a+1]++
	}
	for i := 0; i < n; i++ {
		s.rowPtr[i+1] += s.rowPtr[i]
	}
	// exclusive-topology domain = group of the closest tier; unlabeled nodes get a domain of their own
	domID := map[string]int32{}
	s.domain = make([]int32, n)
	s.free = make([]int32, n)
	for i, nm := range names {
		ni := nc.nodes[nm]
		key, ok := ni.labels[TierLabels[0]]
		if !ok {
			key = "node/" + nm
		}
		id, seen := domID[key]
		if !seen {
			id = int32(len(s.domains))
			domID[key] = id
			s.domains = append(s.domains, key)
		}
		s.domain[i] = id
		s.free[i] = freeSlots(ni)
	}
	s.owner = make([]int32, max(1, len(s.domains)))
	for i := range s.owner {
		s.owner[i] = -1
	}
	for d, gid := range nc.domainOwner {
		if id, ok := domID[d]; ok {
			s.owner[id] = gid
		}
	}
	return s
}

// sync pushes what changed since the last call and returns the snapshot the blob must be built
// against.  Topology change: full upload.  Capacity churn: the incremental refresh when few nodes
// changed (rbgtopo_update_nodes_delta recomputes `base` on their closed neighbourhoods only and
// repairs the background order by merging), else the full refresh.
func (nc *nodeCache) sync(p *placer) (*snapshot, error) {
	nc.mu.Lock()
	defer nc.mu.Unlock()
	if nc.snap == nil || nc.pushedTopo != nc.topoGen {
		s := nc.build()
		if err := p.setTopology(s); err != nil {
			return nil, err
		}
		if nc.classKeys != nil { // set_topology dropped the classes: install those of the new node set
			cls, err := buildNodeClasses(s.names, nc.nodes, nc.classKeys)
			if err != nil {
				return nil, err
			}
			if err := p.setNodeClasses(len(cls.labels), cls.class, nc.topoGen); err != nil {
				return nil, err
			}
			s.classes = cls
		}
		nc.snap, nc.pushedTopo, nc.pushedCap = s, nc.topoGen, nc.capGen
		nc.dirty = map[string]struct{}{}
		return s, nil
	}
	if nc.pushedCap != nc.capGen {
		s := nc.snap
		free := append([]int32(nil), s.free...) // snapshots are immutable: concurrent reconciles read the old one
		var ids, vals []int32
		for nm := range nc.dirty {
			if id, ok := s.ids[nm]; ok {
				free[id] = freeSlots(nc.nodes[nm])
				ids = append(ids, id)
				vals = append(vals, free[id])
			}
		}
		var err error
		if len(ids)*8 <= len(free) {
			err = p.updateNodesDelta(ids, vals, nc.capGen)
		} else {
			err = p.updateNodes(free, nil, nc.capGen)
		}
		if err != nil {
			return nil, err
		}
		ns := *s
		ns.free, ns.capGen = free, nc.capGen
		nc.snap, nc.pushedCap = &ns, nc.capGen
		nc.dirty = map[string]struct{}{}
	}
	return nc.snap, nil
}

// classChanged: a class key's label value or the node's hard taints changed (node eligibility on): the classes are
// rebuilt with the topology.
func (nc *nodeCache) classChanged(old, ni *nodeInfo) bool {
	if nc.classKeys == nil {
		return false
	}
	for _, k := range nc.classKeys {
		if old.labels[k] != ni.labels[k] {
			return true
		}
	}
	a, b := hardTaints(old.taints), hardTaints(ni.taints)
	if len(a) != len(b) {
		return true
	}
	for i := range a {
		if a[i] != b[i] {
			return true
		}
	}
	return false
}
