// Package kgpuscheduler: cgo binding of include/kgpu.h.  UNCOMPILED (no Go toolchain here).
package kgpuscheduler

/*
#cgo CFLAGS: -I${SRCDIR}/../../include
#cgo LDFLAGS: -L${SRCDIR}/../../kubegpu_b200/lib -lkgpu
#include <stdlib.h>
#include "kgpu.h"
*/
import "C"

import (
	"fmt"
	"unsafe"
)

// NoFit mirrors KGPU_NO_FIT.
const NoFit = ^uint64(0)

type handle struct{ h *C.kgpu_t }

func create(devs []int32) (*handle, error) {
	var h *C.kgpu_t
	if rc := C.kgpu_create((*C.int)(unsafe.Pointer(&devs[0])), C.int(len(devs)), &h); rc != C.KGPU_OK {
		return nil, fmt.Errorf("kgpu_create: %s", C.GoString(C.kgpu_last_error(nil)))
	}
	return &handle{h}, nil
}

func (k *handle) destroy() { C.kgpu_destroy(k.h) }

func (k *handle) err(what string) error {
	return fmt.Errorf("%s: %s", what, C.GoString(C.kgpu_last_error(k.h)))
}

// uploadNodes: topo is N*64 int32, free is N int32.  The slices are only borrowed for the
// duration of the call (cgo pointer rule); libkgpu copies them to the device before returning.
func (k *handle) uploadNodes(topo, free []int32, base int64) error {
	if len(free) == 0 {
		if rc := C.kgpu_upload_nodes(k.h, nil, nil, 0, C.int64_t(base)); rc != C.KGPU_OK {
			return k.err("kgpu_upload_nodes")
		}
		return nil
	}
	if rc := C.kgpu_upload_nodes(k.h, (*C.int32_t)(unsafe.Pointer(&topo[0])),
		(*C.int32_t)(unsafe.Pointer(&free[0])), C.int64_t(len(free)), C.int64_t(base)); rc != C.KGPU_OK {
		return k.err("kgpu_upload_nodes")
	}
	return nil
}

func (k *handle) updateNode(idx int64, topo *[64]int32, free int32) error {
	if rc := C.kgpu_update_node(k.h, C.int64_t(idx), (*C.int32_t)(unsafe.Pointer(&topo[0])), C.int32_t(free)); rc != C.KGPU_OK {
		return k.err("kgpu_update_node")
	}
	return nil
}

func (k *handle) setFreeMask(idx int64, free int32) error {
	if rc := C.kgpu_set_free_mask(k.h, C.int64_t(idx), C.int32_t(free)); rc != C.KGPU_OK {
		return k.err("kgpu_set_free_mask")
	}
	return nil
}

// setFreeMasks: a cycle's Take/Return in ONE call (one H2D copy + one kernel on the device).
func (k *handle) setFreeMasks(idx []int64, free []int32) error {
	if len(idx) == 0 {
		return nil
	}
	if rc := C.kgpu_set_free_masks(k.h, (*C.int64_t)(unsafe.Pointer(&idx[0])), (*C.int32_t)(unsafe.Pointer(&free[0])),
		C.int64_t(len(idx))); rc != C.KGPU_OK {
		return k.err("kgpu_set_free_masks")
	}
	return nil
}

// fitLookup: (cost<<8 | mask) of one node for one GPU count from the handle's host-side (node, k)
// table -- no launch, no copy: this is what PodFitsDevice calls once per (node, pod) pair.
func (k *handle) fitLookup(node int64, gpus int32) (uint32, error) {
	var out C.uint32_t
	if rc := C.kgpu_fit_lookup(k.h, C.int64_t(node), C.int32_t(gpus), &out); rc != C.KGPU_OK {
		return 0, k.err("kgpu_fit_lookup")
	}
	return uint32(out), nil
}

// scoreBatch: pods is P*4 int32 {k, pod_id, flags, reserved}; returns P keys
// (cost<<40 | node<<8 | mask) or NoFit.
func (k *handle) scoreBatch(pods []int32) ([]uint64, error) {
	keys := make([]uint64, len(pods)/4)
	if len(keys) == 0 {
		return keys, nil
	}
	if rc := C.kgpu_score_batch(k.h, (*C.int32_t)(unsafe.Pointer(&pods[0])), C.int64_t(len(keys)),
		(*C.uint64_t)(unsafe.Pointer(&keys[0]))); rc != C.KGPU_OK {
		return nil, k.err("kgpu_score_batch")
	}
	return keys, nil
}

// scorePair: (cost<<8 | mask) of one node for one GPU count, or 0xFFFFFFFF.
func (k *handle) scorePair(node int64, gpus int32) (uint32, error) {
	var out C.uint32_t
	n, kk := C.int64_t(node), C.int32_t(gpus)
	if rc := C.kgpu_score_pairs(k.h, &n, &kk, nil, 1, &out); rc != C.KGPU_OK {
		return 0, k.err("kgpu_score_pairs")
	}
	return uint32(out), nil
}

// placeBatch: stateful sequential placement (pods in order, the device-side free masks are
// updated).  dryRun: conflict-free proposals on a scratch copy of the masks, nothing is taken.
// gang: nil, or one id per pod (0 = on its own; a run of consecutive pods with the same nonzero
// id is placed all or nothing, kgpu_place_batch_gang).  Same buffers as scoreBatch.
func (k *handle) placeBatch(pods []int32, gang []int32, dryRun bool) ([]uint64, error) {
	keys := make([]uint64, len(pods)/4)
	if len(keys) == 0 {
		return keys, nil
	}
	flags := C.int(0)
	if dryRun {
		flags = C.KGPU_PLACE_DRY_RUN
	}
	var g *C.int32_t
	if gang != nil {
		g = (*C.int32_t)(unsafe.Pointer(&gang[0]))
	}
	if rc := C.kgpu_place_batch_gang(k.h, (*C.int32_t)(unsafe.Pointer(&pods[0])), g, C.int64_t(len(keys)),
		(*C.uint64_t)(unsafe.Pointer(&keys[0])), flags); rc != C.KGPU_OK {
		return nil, k.err("kgpu_place_batch_gang")
	}
	return keys, nil
}

// uploadDomains: each node's network domain, -1 (none) or 0..n-1 (kgpu_upload_domains); len(domain) = the node count.
func (k *handle) uploadDomains(domain []int32) error {
	var d *C.int32_t
	if len(domain) > 0 {
		d = (*C.int32_t)(unsafe.Pointer(&domain[0]))
	}
	if rc := C.kgpu_upload_domains(k.h, d, C.int64_t(len(domain))); rc != C.KGPU_OK {
		return k.err("kgpu_upload_domains")
	}
	return nil
}

// placeBatchDomain: placeBatch with one gang_domain value per pod (kgpu_place_batch_gang_domain): 0 = no constraint,
// C.KGPU_GANG_DOMAIN_REQUIRED = the gang inside one domain or not at all, C.KGPU_GANG_DOMAIN_PREFERRED = inside one
// domain if one fits, else as a plain gang.  gangDomain nil is placeBatch.
func (k *handle) placeBatchDomain(pods []int32, gang []int32, gangDomain []int32, dryRun bool) ([]uint64, error) {
	keys := make([]uint64, len(pods)/4)
	if len(keys) == 0 {
		return keys, nil
	}
	flags := C.int(0)
	if dryRun {
		flags = C.KGPU_PLACE_DRY_RUN
	}
	var g, gd *C.int32_t
	if gang != nil {
		g = (*C.int32_t)(unsafe.Pointer(&gang[0]))
	}
	if gangDomain != nil {
		gd = (*C.int32_t)(unsafe.Pointer(&gangDomain[0]))
	}
	if rc := C.kgpu_place_batch_gang_domain(k.h, (*C.int32_t)(unsafe.Pointer(&pods[0])), g, gd, C.int64_t(len(keys)),
		(*C.uint64_t)(unsafe.Pointer(&keys[0])), flags); rc != C.KGPU_OK {
		return nil, k.err("kgpu_place_batch_gang_domain")
	}
	return keys, nil
}

// uploadDomainLevels: nested network domains (kgpu_upload_domain_levels), domain[l][i] = node i's domain at level l
// (level 0 the finest), -1 or 0..n-1; every level holds the node count, the levels nest, 1..C.KGPU_MAX_DOMAIN_LEVELS
// levels.
func (k *handle) uploadDomainLevels(domain [][]int32) error {
	if len(domain) == 0 {
		return k.uploadDomains(nil)
	}
	n := len(domain[0])
	flat := make([]int32, 0, len(domain)*n)
	for _, lv := range domain {
		if len(lv) != n {
			return fmt.Errorf("uploadDomainLevels: levels of different lengths")
		}
		flat = append(flat, lv...)
	}
	var d *C.int32_t
	if len(flat) > 0 {
		d = (*C.int32_t)(unsafe.Pointer(&flat[0]))
	}
	if rc := C.kgpu_upload_domain_levels(k.h, d, C.int(len(domain)), C.int64_t(n)); rc != C.KGPU_OK {
		return k.err("kgpu_upload_domain_levels")
	}
	return nil
}

// placeBatchLevels: placeBatchDomain with one gang_level per pod (kgpu_place_batch_gang_levels): the highest level a
// constrained gang may span; the gang takes the lowest level 0..gang_level with a fitting domain.  gangLevel nil is
// placeBatchDomain.
func (k *handle) placeBatchLevels(pods []int32, gang []int32, gangDomain []int32, gangLevel []int32, dryRun bool) ([]uint64, error) {
	keys := make([]uint64, len(pods)/4)
	if len(keys) == 0 {
		return keys, nil
	}
	flags := C.int(0)
	if dryRun {
		flags = C.KGPU_PLACE_DRY_RUN
	}
	var g, gd, gl *C.int32_t
	if gang != nil {
		g = (*C.int32_t)(unsafe.Pointer(&gang[0]))
	}
	if gangDomain != nil {
		gd = (*C.int32_t)(unsafe.Pointer(&gangDomain[0]))
	}
	if gangLevel != nil {
		gl = (*C.int32_t)(unsafe.Pointer(&gangLevel[0]))
	}
	if rc := C.kgpu_place_batch_gang_levels(k.h, (*C.int32_t)(unsafe.Pointer(&pods[0])), g, gd, gl, C.int64_t(len(keys)),
		(*C.uint64_t)(unsafe.Pointer(&keys[0])), flags); rc != C.KGPU_OK {
		return nil, k.err("kgpu_place_batch_gang_levels")
	}
	return keys, nil
}

func (k *handle) freeMasks(n int64) ([]int32, error) {
	out := make([]int32, n)
	if n == 0 {
		return out, nil
	}
	if rc := C.kgpu_get_free_masks(k.h, (*C.int32_t)(unsafe.Pointer(&out[0])), C.int64_t(n)); rc != C.KGPU_OK {
		return nil, k.err("kgpu_get_free_masks")
	}
	return out, nil
}

// uploadHolders: the whole holder table, 8 entries per node (-1, or level<<3 | owner), n = the node count.
func (k *handle) uploadHolders(holders []int32) error {
	n := len(holders) / 8
	var p *C.int32_t
	if n > 0 {
		p = (*C.int32_t)(unsafe.Pointer(&holders[0]))
	}
	if rc := C.kgpu_upload_holders(k.h, p, C.int64_t(n)); rc != C.KGPU_OK {
		return k.err("kgpu_upload_holders")
	}
	return nil
}

// setHolders: replace the rows of nodes idx (holders holds 8 entries per index) in one copy; the last row wins.
func (k *handle) setHolders(idx []int64, holders []int32) error {
	if len(idx) == 0 {
		return nil
	}
	if rc := C.kgpu_set_holders(k.h, (*C.int64_t)(unsafe.Pointer(&idx[0])), (*C.int32_t)(unsafe.Pointer(&holders[0])),
		C.int64_t(len(idx))); rc != C.KGPU_OK {
		return k.err("kgpu_set_holders")
	}
	return nil
}

// preemptBatch: for each pod the best placement when running pods of a lower level (lvl, 0..15) may be evicted,
// and the owner mask of its victims on the key's node (kgpu_preempt_batch).  Same pod buffer as scoreBatch.
func (k *handle) preemptBatch(pods []int32, lvl []int32) ([]uint64, []uint32, error) {
	keys := make([]uint64, len(pods)/4)
	victims := make([]uint32, len(keys))
	if len(keys) == 0 {
		return keys, victims, nil
	}
	if rc := C.kgpu_preempt_batch(k.h, (*C.int32_t)(unsafe.Pointer(&pods[0])), (*C.int32_t)(unsafe.Pointer(&lvl[0])),
		C.int64_t(len(keys)), (*C.uint64_t)(unsafe.Pointer(&keys[0])), (*C.uint32_t)(unsafe.Pointer(&victims[0]))); rc != C.KGPU_OK {
		return nil, nil, k.err("kgpu_preempt_batch")
	}
	return keys, victims, nil
}

// preemptPlan: preemptBatch taken in order (kgpu_preempt_plan): each pod sees the GPUs the pods before it take and the
// GPUs their victims free, and no two pods name the same victim.  Dry run: commit with setFreeMasks / setHolders once
// the victims are gone.
func (k *handle) preemptPlan(pods []int32, lvl []int32) ([]uint64, []uint32, error) {
	keys := make([]uint64, len(pods)/4)
	victims := make([]uint32, len(keys))
	if len(keys) == 0 {
		return keys, victims, nil
	}
	if rc := C.kgpu_preempt_plan(k.h, (*C.int32_t)(unsafe.Pointer(&pods[0])), (*C.int32_t)(unsafe.Pointer(&lvl[0])),
		C.int64_t(len(keys)), (*C.uint64_t)(unsafe.Pointer(&keys[0])), (*C.uint32_t)(unsafe.Pointer(&victims[0]))); rc != C.KGPU_OK {
		return nil, nil, k.err("kgpu_preempt_plan")
	}
	return keys, victims, nil
}

// preemptPlanGang: preemptPlan with gang ids (kgpu_preempt_plan_gang, ids as for placeBatch): a gang's members
// evict and take all together or not at all, and a failed gang's would-be victims stay available to later pods.
func (k *handle) preemptPlanGang(pods []int32, lvl []int32, gang []int32) ([]uint64, []uint32, error) {
	keys := make([]uint64, len(pods)/4)
	victims := make([]uint32, len(keys))
	if len(keys) == 0 {
		return keys, victims, nil
	}
	if rc := C.kgpu_preempt_plan_gang(k.h, (*C.int32_t)(unsafe.Pointer(&pods[0])), (*C.int32_t)(unsafe.Pointer(&lvl[0])),
		(*C.int32_t)(unsafe.Pointer(&gang[0])), C.int64_t(len(keys)), (*C.uint64_t)(unsafe.Pointer(&keys[0])),
		(*C.uint32_t)(unsafe.Pointer(&victims[0]))); rc != C.KGPU_OK {
		return nil, nil, k.err("kgpu_preempt_plan_gang")
	}
	return keys, victims, nil
}

// preemptPlanDomain: preemptPlanGang with gang domains (kgpu_preempt_plan_gang_domain, gangDomain as for
// placeBatchDomain): a REQUIRED gang evicts and takes its GPUs inside one domain of uploadDomains or gets NO_FIT; a
// PREFERRED gang falls back to the plain gang plan.  gang may be nil when every gangDomain value is 0.
func (k *handle) preemptPlanDomain(pods []int32, lvl []int32, gang []int32, gangDomain []int32) ([]uint64, []uint32, error) {
	keys := make([]uint64, len(pods)/4)
	victims := make([]uint32, len(keys))
	if len(keys) == 0 {
		return keys, victims, nil
	}
	var g, gd *C.int32_t
	if gang != nil {
		g = (*C.int32_t)(unsafe.Pointer(&gang[0]))
	}
	if gangDomain != nil {
		gd = (*C.int32_t)(unsafe.Pointer(&gangDomain[0]))
	}
	if rc := C.kgpu_preempt_plan_gang_domain(k.h, (*C.int32_t)(unsafe.Pointer(&pods[0])), (*C.int32_t)(unsafe.Pointer(&lvl[0])), g, gd,
		C.int64_t(len(keys)), (*C.uint64_t)(unsafe.Pointer(&keys[0])), (*C.uint32_t)(unsafe.Pointer(&victims[0]))); rc != C.KGPU_OK {
		return nil, nil, k.err("kgpu_preempt_plan_gang_domain")
	}
	return keys, victims, nil
}
