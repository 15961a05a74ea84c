/*
Copyright 2024 The RoleBasedGroup Authors.

Licensed under the Apache License, Version 2.0 (the "License").
*/

// cgo binding of include/rbgtopo.h (librbgtopo.so).
//
// NOT COMPILED IN THE BUILD IMAGE OF THIS REPO (no Go toolchain there): source for a maintainer.
// tests/cabi_driver.c calls the same entry points with the same plain-C argument shapes from ten
// pthreads, which is what these wrappers do from ten goroutines.
//
// Error text and goroutine migration: rbgtopo_last_error returns the calling THREAD's last error.
// A goroutine can move to another OS thread between two cgo calls, so every wrapper below makes
// the call AND fetches the error text inside ONE C helper (rbgtopo_go_*): no Go scheduling point
// lies in between, no runtime.LockOSThread is needed.
package b200topo

/*
#cgo CFLAGS: -I${SRCDIR}/../../../third_party/rbgtopo/include
#cgo LDFLAGS: -L${SRCDIR}/../../../third_party/rbgtopo/lib -lrbgtopo -lcudart
#include <stdlib.h>
#include <string.h>
#include "rbgtopo.h"

#define RBGTOPO_GO_ERRLEN 512

static void rbgtopo_go_err(rbgtopo_ctx* ctx, int32_t rc, char* err) {
  if (rc != RBGTOPO_OK) rbgtopo_last_error(ctx, err, RBGTOPO_GO_ERRLEN); else err[0] = 0;
}
static int32_t rbgtopo_go_create(int32_t device, int32_t rank, int32_t world, rbgtopo_ctx** out, char* err) {
  rbgtopo_config cfg;
  memset(&cfg, 0, sizeof cfg);
  cfg.device = device; cfg.rank = rank; cfg.world = world;
  int32_t rc = rbgtopo_create(&cfg, out);
  rbgtopo_go_err(NULL, rc, err);
  return rc;
}
static int32_t rbgtopo_go_set_topology(rbgtopo_ctx* ctx, int32_t n, int64_t e, const int32_t* row_ptr, const int32_t* col,
                                       const int32_t* w, const int32_t* free_slots, const int32_t* domain,
                                       int32_t n_domains, const int32_t* owner, uint64_t gen, char* err) {
  int32_t rc = rbgtopo_set_topology(ctx, n, e, row_ptr, col, w, free_slots, domain, n_domains, owner, gen);
  rbgtopo_go_err(ctx, rc, err);
  return rc;
}
static int32_t rbgtopo_go_update_nodes(rbgtopo_ctx* ctx, const int32_t* free_slots, const int32_t* owner, uint64_t gen,
                                       char* err) {
  int32_t rc = rbgtopo_update_nodes(ctx, free_slots, owner, gen);
  rbgtopo_go_err(ctx, rc, err);
  return rc;
}
static int32_t rbgtopo_go_update_nodes_delta(rbgtopo_ctx* ctx, int32_t n_changed, const int32_t* nodes,
                                             const int32_t* free_slots, uint64_t gen, char* err) {
  int32_t rc = rbgtopo_update_nodes_delta(ctx, n_changed, nodes, free_slots, gen);
  rbgtopo_go_err(ctx, rc, err);
  return rc;
}
static int32_t rbgtopo_go_set_exclusive_levels(rbgtopo_ctx* ctx, int32_t n_levels, const int32_t* level_domain,
                                              const int32_t* level_n_domains, int32_t n_occ, const int32_t* occ,
                                              uint64_t gen, char* err) {
  int32_t rc = rbgtopo_set_exclusive_levels(ctx, n_levels, level_domain, level_n_domains, n_occ, occ, gen);
  rbgtopo_go_err(ctx, rc, err);
  return rc;
}
static int32_t rbgtopo_go_place_groups(rbgtopo_ctx* ctx, const int32_t* groups, int64_t words, int32_t* assign,
                                       int32_t* status, int32_t* domain, char* err) {
  int32_t rc = rbgtopo_place_groups(ctx, groups, words, assign, status, domain);
  rbgtopo_go_err(ctx, rc, err);
  return rc;
}
static int32_t rbgtopo_go_place_groups_committed(rbgtopo_ctx* ctx, const int32_t* groups, int64_t words,
                                                 int32_t* assign, int32_t* status, int32_t* domain, int32_t* rounds,
                                                 char* err) {
  int32_t rc = rbgtopo_place_groups_committed(ctx, groups, words, assign, status, domain, rounds);
  rbgtopo_go_err(ctx, rc, err);
  return rc;
}
static int32_t rbgtopo_go_place_groups_ranked(rbgtopo_ctx* ctx, const int32_t* groups, int64_t words, int32_t n_alt,
                                              int32_t* assign, int32_t* status, int32_t* domain, float* score,
                                              int32_t* alt_node, float* alt_score, char* err) {
  int32_t rc = rbgtopo_place_groups_ranked(ctx, groups, words, n_alt, assign, status, domain, score, alt_node, alt_score);
  rbgtopo_go_err(ctx, rc, err);
  return rc;
}
*/
import "C"

import (
	"fmt"
	"unsafe"
)

// Status codes of include/rbgtopo.h the shim distinguishes.
const (
	codeOK       = int32(C.RBGTOPO_OK)
	codeInvalid  = int32(C.RBGTOPO_EINVAL)
	codeNoDevice = int32(C.RBGTOPO_ENODEVICE)
	codeCUDA     = int32(C.RBGTOPO_ECUDA)
	codeInexact  = int32(C.RBGTOPO_EINEXACT)
	codeLimit    = int32(C.RBGTOPO_ELIMIT)
)

// placerError carries the library's status code so that the manager can tell "bad input"
// (report) from "device trouble" (degrade to no placement hint, SURVEY.md §8b "Errors").
type placerError struct {
	code int32
	text string
}

func (e *placerError) Error() string { return fmt.Sprintf("rbgtopo error %d: %s", e.code, e.text) }

// deviceTrouble: the controller must keep working exactly as it does today (no hint), not requeue forever.
func (e *placerError) deviceTrouble() bool { return e.code == codeCUDA || e.code == codeNoDevice }

func p32(s []int32) *C.int32_t {
	if len(s) == 0 {
		return nil
	}
	return (*C.int32_t)(unsafe.Pointer(&s[0]))
}

func mkErr(rc C.int32_t, buf *[C.RBGTOPO_GO_ERRLEN]C.char) error {
	if rc == C.RBGTOPO_OK {
		return nil
	}
	return &placerError{code: int32(rc), text: C.GoString(&buf[0])}
}

// placer owns one rbgtopo_ctx (device memory, streams, staging).  All methods are safe for
// concurrent use by --max-concurrent-reconciles goroutines (cmd/rbgs/main.go:140-143): the library
// takes an internal slot per call (include/rbgtopo.h, "Rules of the ABI").
type placer struct {
	ctx *C.rbgtopo_ctx
}

func newPlacer(device int) (*placer, error) {
	var buf [C.RBGTOPO_GO_ERRLEN]C.char
	p := &placer{}
	rc := C.rbgtopo_go_create(C.int32_t(device), 0, 1, &p.ctx, &buf[0])
	if err := mkErr(rc, &buf); err != nil {
		return nil, err
	}
	return p, nil
}

func (p *placer) close() {
	if p != nil && p.ctx != nil {
		C.rbgtopo_destroy(p.ctx)
		p.ctx = nil
	}
}

// Every slice is plain int32 without Go pointers inside and is only read during the call: the
// library copies into pinned staging before returning (cgo pointer-passing rules).
func (p *placer) setTopology(s *snapshot) error {
	var buf [C.RBGTOPO_GO_ERRLEN]C.char
	rc := C.rbgtopo_go_set_topology(p.ctx, C.int32_t(len(s.names)), C.int64_t(len(s.colIdx)), p32(s.rowPtr), p32(s.colIdx),
		p32(s.edgeW), p32(s.free), p32(s.domain), C.int32_t(len(s.owner)), p32(s.owner), C.uint64_t(s.topoGen), &buf[0])
	return mkErr(rc, &buf)
}

func (p *placer) updateNodes(free, owner []int32, gen uint64) error {
	var buf [C.RBGTOPO_GO_ERRLEN]C.char
	rc := C.rbgtopo_go_update_nodes(p.ctx, p32(free), p32(owner), C.uint64_t(gen), &buf[0])
	return mkErr(rc, &buf)
}

// updateNodesDelta: capacity of a few nodes changed (pod bound / deleted): incremental refresh of
// base / order on the device (rbgtopo_update_nodes_delta, SURVEY.md §8f rank 3).
func (p *placer) updateNodesDelta(nodes, free []int32, gen uint64) error {
	var buf [C.RBGTOPO_GO_ERRLEN]C.char
	rc := C.rbgtopo_go_update_nodes_delta(p.ctx, C.int32_t(len(nodes)), p32(nodes), p32(free), C.uint64_t(gen), &buf[0])
	return mkErr(rc, &buf)
}

// setExclusiveLevels: occupancy mode (DESIGN.md §3.9).  levelDomain holds nLevels rows of n node domains (nil keeps
// the installed partitions and refreshes the records only); occ holds (node, gid, level) per pod carrying the
// group-unique-hash label.
func (p *placer) setExclusiveLevels(nLevels int, levelDomain, levelNDomains, occ []int32, gen uint64) error {
	var buf [C.RBGTOPO_GO_ERRLEN]C.char
	rc := C.rbgtopo_go_set_exclusive_levels(p.ctx, C.int32_t(nLevels), p32(levelDomain), p32(levelNDomains),
		C.int32_t(len(occ)/3), p32(occ), C.uint64_t(gen), &buf[0])
	return mkErr(rc, &buf)
}

// placeGroups: one GROUPS blob in, (assign per pending replica, status and exclusive domain per group) out.
func (p *placer) placeGroups(blob []int32) (assign, status, domain []int32, err error) {
	nGroups, nPending := int(blob[2]), int(blob[4])
	assign = make([]int32, max(nPending, 1))
	status = make([]int32, max(nGroups, 1))
	domain = make([]int32, max(nGroups, 1))
	var buf [C.RBGTOPO_GO_ERRLEN]C.char
	rc := C.rbgtopo_go_place_groups(p.ctx, p32(blob), C.int64_t(len(blob)), p32(assign), p32(status), p32(domain), &buf[0])
	if err = mkErr(rc, &buf); err != nil {
		return nil, nil, nil, err
	}
	return assign[:nPending], status[:nGroups], domain[:nGroups], nil
}

// placeGroupsCommitted: placeGroups as a committed batch (DESIGN.md §3.8): the groups in blob order, each seeing the
// capacity and exclusive domains the groups before it took; rounds = selection rounds the library ran.
func (p *placer) placeGroupsCommitted(blob []int32) (assign, status, domain []int32, rounds int32, err error) {
	nGroups, nPending := int(blob[2]), int(blob[4])
	assign = make([]int32, max(nPending, 1))
	status = make([]int32, max(nGroups, 1))
	domain = make([]int32, max(nGroups, 1))
	var r C.int32_t
	var buf [C.RBGTOPO_GO_ERRLEN]C.char
	rc := C.rbgtopo_go_place_groups_committed(p.ctx, p32(blob), C.int64_t(len(blob)), p32(assign), p32(status), p32(domain),
		&r, &buf[0])
	if err = mkErr(rc, &buf); err != nil {
		return nil, nil, nil, 0, err
	}
	return assign[:nPending], status[:nGroups], domain[:nGroups], int32(r), nil
}

// placeGroupsRanked: placeGroups plus, per pending replica, up to nAlt next-best nodes that still have room once its
// group is placed (DESIGN.md §3.10); altNode[r*nAlt+i] = -1 where there are fewer.  assign / status / domain are
// placeGroups'.
func (p *placer) placeGroupsRanked(blob []int32, nAlt int) (assign, status, domain, altNode []int32, err error) {
	nGroups, nPending := int(blob[2]), int(blob[4])
	assign = make([]int32, max(nPending, 1))
	status = make([]int32, max(nGroups, 1))
	domain = make([]int32, max(nGroups, 1))
	score := make([]float32, max(nPending, 1))
	altNode = make([]int32, max(nPending*nAlt, 1))
	altScore := make([]float32, max(nPending*nAlt, 1))
	var buf [C.RBGTOPO_GO_ERRLEN]C.char
	rc := C.rbgtopo_go_place_groups_ranked(p.ctx, p32(blob), C.int64_t(len(blob)), C.int32_t(nAlt), p32(assign), p32(status),
		p32(domain), (*C.float)(unsafe.Pointer(&score[0])), p32(altNode), (*C.float)(unsafe.Pointer(&altScore[0])), &buf[0])
	if err = mkErr(rc, &buf); err != nil {
		return nil, nil, nil, nil, err
	}
	return assign[:nPending], status[:nGroups], domain[:nGroups], altNode[:nPending*nAlt], nil
}
