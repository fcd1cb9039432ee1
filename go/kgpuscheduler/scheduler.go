// UNCOMPILED (no Go toolchain here).  DeviceScheduler over libkgpu with the reference's
// method set (gpuschedulerplugin/gpu_scheduler.go:21-71).  The tree cache / DevRequests rewrite
// is delegated to the reference's own package so the core's group allocator keeps working;
// the score and the placement come from the GPU.
package kgpuscheduler

import (
	"fmt"
	"regexp"
	"sort"
	"sync"

	"github.com/Microsoft/KubeDevice-API/pkg/devicescheduler"
	types "github.com/Microsoft/KubeDevice-API/pkg/types"
	gtype "github.com/Microsoft/KubeGPU/gpuplugintypes"
	ref "github.com/Microsoft/KubeGPU/gpuschedulerplugin"
)

var gpuKey = regexp.MustCompile(string(types.DeviceGroupPrefix) + `/(gpugrp1/(.*?)/gpugrp0/(.*?)/gpu/(.*?))/cards`)

// a DevRequests key that names one GPU card (compiled ONCE: the reference compiles its regexps per call,
// gpu.go:131, which is the per-call cost SURVEY.md 3 criticises)
var gpuCardReq = regexp.MustCompile(`/gpu/.*/cards$`)

type nodeRec struct {
	index   int64
	names   []string // slot -> "gpugrp1/a/gpugrp0/b/gpu/<id>"
	topo    [64]int32
	present uint32
	used    uint32
	removed bool
}

type placement struct {
	node      string
	mask      uint32
	cost      uint32
	committed bool // the GPUs are already taken on the device (PlaceBatch) or by TakePodResources
}

// NvidiaGPUScheduler implements devicescheduler.DeviceScheduler.
type NvidiaGPUScheduler struct {
	mu     sync.Mutex
	h      *handle
	nodes  map[string]*nodeRec
	byIdx  []string
	dirty   bool            // node COUNT changed: re-upload
	changed map[string]bool // existing nodes whose matrix / presence changed: kgpu_update_node each
	placed  map[string]placement // pod name -> last placement
	// GroupSchedulerMode false (default): the plugin's (node, GPU set) is authoritative: PodAllocate fills
	// AllocateFrom and UsingGroupScheduler() returns false.  true: the reference's contract
	// (gpu_scheduler.go:69-71): DevRequests only, the core's group allocator does the rest.
	GroupSchedulerMode bool
}

// New creates the scheduler on the given CUDA devices (one handle shards over all of them).
func New(devs []int32) (*NvidiaGPUScheduler, error) {
	h, err := create(devs)
	if err != nil {
		return nil, err
	}
	return &NvidiaGPUScheduler{h: h, nodes: map[string]*nodeRec{}, changed: map[string]bool{}, placed: map[string]placement{}}, nil
}

func level(a, b []string) int32 { // same gpugrp0 -> 5, same gpugrp1 -> 3, else 1
	if a[2] == b[2] && a[3] == b[3] {
		return 5
	}
	if a[2] == b[2] {
		return 3
	}
	return 1
}

func (ns *NvidiaGPUScheduler) AddNode(nodeName string, nodeInfo *types.NodeInfo) {
	(&ref.NvidiaGPUScheduler{}).AddNode(nodeName, nodeInfo) // translation + tree cache, gpu_scheduler.go:21-28
	ns.mu.Lock()
	defer ns.mu.Unlock()
	keys := make([]string, 0, len(nodeInfo.Allocatable))
	for k := range nodeInfo.Allocatable {
		keys = append(keys, string(k))
	}
	sort.Strings(keys)
	var slots [][]string
	for _, k := range keys {
		if m := gpuKey.FindStringSubmatch(k); len(m) == 5 && len(slots) < 8 {
			slots = append(slots, m)
		}
	}
	rec, ok := ns.nodes[nodeName]
	if !ok {
		rec = &nodeRec{index: int64(len(ns.byIdx))}
		ns.nodes[nodeName] = rec
		ns.byIdx = append(ns.byIdx, nodeName)
		ns.dirty = true
	} else {
		ns.changed[nodeName] = true
	}
	rec.removed, rec.names, rec.topo = false, nil, [64]int32{}
	for i, a := range slots {
		rec.names = append(rec.names, a[1])
		for j, b := range slots {
			if i != j {
				rec.topo[i*8+j] = level(a, b)
			}
		}
	}
	rec.present = uint32(1)<<uint(len(slots)) - 1
}

func (ns *NvidiaGPUScheduler) RemoveNode(nodeName string) {
	(&ref.NvidiaGPUScheduler{}).RemoveNode(nodeName)
	ns.mu.Lock()
	defer ns.mu.Unlock()
	if rec, ok := ns.nodes[nodeName]; ok {
		rec.removed = true
		ns.changed[nodeName] = true
	}
}

func freeOf(rec *nodeRec) int32 {
	if rec.removed {
		return 0
	}
	return int32(rec.present &^ rec.used)
}

func (ns *NvidiaGPUScheduler) flush() error {
	if !ns.dirty {
		// only existing nodes changed: one 256-byte update each instead of re-uploading the cluster
		for name := range ns.changed {
			rec := ns.nodes[name]
			if err := ns.h.updateNode(rec.index, &rec.topo, freeOf(rec)); err != nil {
				return err
			}
		}
		ns.changed = map[string]bool{}
		return nil
	}
	ns.changed = map[string]bool{}
	topo := make([]int32, 64*len(ns.byIdx))
	free := make([]int32, len(ns.byIdx))
	for i, name := range ns.byIdx {
		rec := ns.nodes[name]
		copy(topo[64*i:], rec.topo[:])
		if !rec.removed {
			free[i] = int32(rec.present &^ rec.used)
		}
	}
	if err := ns.h.uploadNodes(topo, free, 0); err != nil {
		return err
	}
	ns.dirty = false
	return nil
}

func podGPUs(podInfo *types.PodInfo) int32 { // gpu.go:295-303
	n := int64(0)
	for _, c := range podInfo.RunningContainers {
		n += c.Requests[gtype.ResourceGPU]
	}
	for _, c := range podInfo.InitContainers {
		if c.Requests[gtype.ResourceGPU] > n {
			n = c.Requests[gtype.ResourceGPU]
		}
	}
	if n > 8 {
		n = 9
	}
	return int32(n)
}

// GPUGangID: pod-level request (extension); pods of one PlaceBatch / ProposeBatch with the same nonzero value are
// placed all or nothing.  ScoreBatch ignores it: snapshot scores change no state.
const GPUGangID = "gpu/gpu-gang-id"

// gangOrder: the device takes a gang as one run of consecutive pods with an int32 id, so ids are renumbered 1, 2, ...
// in order of first appearance and each member moves up to its gang's first member.  order[i] = the caller's index of
// the pod at device position i; gang is nil when no pod carries an id.
func gangOrder(pods []*types.PodInfo) (order []int, gang []int32) {
	dense := map[int64]int32{}
	var members [][]int
	of := make([]int32, len(pods))
	for i, p := range pods {
		id := p.Requests[GPUGangID]
		if id == 0 {
			continue
		}
		g, ok := dense[id]
		if !ok {
			g = int32(len(members) + 1)
			dense[id] = g
			members = append(members, nil)
		}
		of[i] = g
		members[g-1] = append(members[g-1], i)
	}
	order = make([]int, 0, len(pods))
	if len(members) == 0 {
		for i := range pods {
			order = append(order, i)
		}
		return order, nil
	}
	gang = make([]int32, 0, len(pods))
	done := make([]bool, len(members))
	for i := range pods {
		switch g := of[i]; {
		case g == 0:
			order, gang = append(order, i), append(gang, 0)
		case !done[g-1]:
			done[g-1] = true
			for _, m := range members[g-1] {
				order, gang = append(order, m), append(gang, g)
			}
		}
	}
	return order, gang
}

func (ns *NvidiaGPUScheduler) runBatch(pods []*types.PodInfo, mode int) ([]uint64, error) { // 0 snapshot, 1 sequential, 2 dry run
	ns.mu.Lock()
	defer ns.mu.Unlock()
	if err := ns.flush(); err != nil {
		return nil, err
	}
	order, gang := gangOrder(pods)
	if mode == 0 {
		for i := range order {
			order[i] = i
		}
		gang = nil
	}
	req := make([]int32, 4*len(pods))
	for i, p := range order {
		req[4*i], req[4*i+1] = podGPUs(pods[p]), int32(p)
	}
	var dev []uint64
	var err error
	if mode == 0 {
		dev, err = ns.h.scoreBatch(req)
	} else {
		dev, err = ns.h.placeBatch(req, gang, mode == 2)
	}
	if err != nil {
		return nil, err
	}
	keys := make([]uint64, len(pods)) // back in the caller's order
	for i, p := range order {
		keys[p] = dev[i]
	}
	for i, p := range pods {
		if keys[i] == NoFit {
			delete(ns.placed, p.Name)
			continue
		}
		pl := placement{ns.byIdx[(keys[i]>>8)&0xFFFFFFFF], uint32(keys[i] & 0xFF), uint32(keys[i] >> 40), mode == 1}
		if mode == 1 { // the device already took them: TakePodResources is a no-op
			ns.nodes[pl.node].used |= pl.mask
		}
		ns.placed[p.Name] = pl
	}
	return keys, nil
}

// ScoreBatch is the batched side door: one kernel launch for a whole scheduling cycle (snapshot scores:
// pods of equal k get the same GPUs -- commit one, re-score the rest, or use ProposeBatch).
func (ns *NvidiaGPUScheduler) ScoreBatch(pods []*types.PodInfo) ([]uint64, error) { return ns.runBatch(pods, 0) }

// PlaceBatch places the cycle in order ON the device: each pod takes its GPUs before the next is scored.
func (ns *NvidiaGPUScheduler) PlaceBatch(pods []*types.PodInfo) ([]uint64, error) { return ns.runBatch(pods, 1) }

// ProposeBatch: conflict-free proposals (PlaceBatch on a scratch copy of the device state); TakePodResources
// commits a pod.
func (ns *NvidiaGPUScheduler) ProposeBatch(pods []*types.PodInfo) ([]uint64, error) { return ns.runBatch(pods, 2) }

// nodeKey: (cost<<8 | mask) of this node for the pod, from the (node, k) fit table (no launch per call).
func (ns *NvidiaGPUScheduler) nodeKey(rec *nodeRec, podInfo *types.PodInfo) (uint32, error) {
	if err := ns.flush(); err != nil {
		return 0, err
	}
	return ns.h.fitLookup(rec.index, podGPUs(podInfo))
}

func (ns *NvidiaGPUScheduler) PodFitsDevice(nodeInfo *types.NodeInfo, podInfo *types.PodInfo, fillAllocateFrom bool) (bool, []devicescheduler.PredicateFailureReason, float64) {
	fits, reasons, _ := (&ref.NvidiaGPUScheduler{}).PodFitsDevice(nodeInfo, podInfo, fillAllocateFrom)
	if !fits {
		return false, reasons, 0.0
	}
	ns.mu.Lock()
	defer ns.mu.Unlock()
	rec, ok := ns.nodes[nodeInfo.Name] // NodeInfo.Name: field of KubeDevice-API's NodeInfo (assumed; the reference never reads it)
	if !ok || rec.removed {
		return true, nil, 0.0 // a node AddNode never saw: the reference's answer
	}
	nk, err := ns.nodeKey(rec, podInfo)
	if err != nil || nk == 0xFFFFFFFF {
		return false, nil, 0.0 // device error or no free GPU set on this node now: does not fit (errors collapse to false, gpu_scheduler.go:35-42)
	}
	if fillAllocateFrom && !ns.GroupSchedulerMode {
		ns.placed[podInfo.Name] = placement{nodeInfo.Name, nk & 0xFF, nk >> 8, false}
	}
	return true, nil, 1.0 / (1.0 + float64(nk>>8))
}

func (ns *NvidiaGPUScheduler) PodAllocate(nodeInfo *types.NodeInfo, podInfo *types.PodInfo) error {
	if err := (&ref.NvidiaGPUScheduler{}).PodAllocate(nodeInfo, podInfo); err != nil {
		return err
	}
	if ns.GroupSchedulerMode {
		return nil // the reference's contract: DevRequests rewritten, AllocateFrom left to the core
	}
	ns.mu.Lock()
	defer ns.mu.Unlock()
	pl, ok := ns.placed[podInfo.Name]
	if here, known := ns.nodes[nodeInfo.Name]; known && (!ok || pl.node != nodeInfo.Name) {
		nk, err := ns.nodeKey(here, podInfo) // no placement recorded for this node: ask the device now
		if err != nil {
			return err
		}
		if nk == 0xFFFFFFFF {
			return fmt.Errorf("PodAllocate: not enough free GPUs on %s", nodeInfo.Name)
		}
		pl, ok = placement{nodeInfo.Name, nk & 0xFF, nk >> 8, false}, true
		ns.placed[podInfo.Name] = pl
	}
	if !ok {
		return nil
	}
	rec := ns.nodes[pl.node]
	var slots []int
	for i := 0; i < 8; i++ {
		if pl.mask>>uint(i)&1 == 1 {
			slots = append(slots, i)
		}
	}
	next := 0
	names := make([]string, 0, len(podInfo.RunningContainers))
	for n := range podInfo.RunningContainers {
		names = append(names, n)
	}
	sort.Strings(names)
	for _, n := range names {
		cont := podInfo.RunningContainers[n]
		cont.AllocateFrom = types.ResourceLocation{}
		reqs := make([]string, 0, len(cont.DevRequests))
		for r := range cont.DevRequests {
			reqs = append(reqs, string(r))
		}
		sort.Strings(reqs)
		for _, r := range reqs {
			if next < len(slots) && gpuCardReq.MatchString(r) {
				cont.AllocateFrom[types.ResourceName(r)] = types.ResourceName(fmt.Sprintf("%s/%s/cards", types.DeviceGroupPrefix, rec.names[slots[next]]))
				next++
			}
		}
		podInfo.RunningContainers[n] = cont
	}
	return nil
}

// take / release: gpu_scheduler.go:57-63 are no-ops in the reference.  Take is idempotent (a placement PlaceBatch
// committed on the device, or one taken before, succeeds without touching anything); GPUs in use by ANOTHER pod
// are an error: score that pod again.
func (ns *NvidiaGPUScheduler) take(podInfo *types.PodInfo, release bool) error {
	ns.mu.Lock()
	defer ns.mu.Unlock()
	pl, ok := ns.placed[podInfo.Name]
	if !ok {
		return nil
	}
	rec := ns.nodes[pl.node]
	if release {
		delete(ns.placed, podInfo.Name)
		if !pl.committed {
			return nil
		}
		rec.used &^= pl.mask
	} else {
		if pl.committed {
			return nil
		}
		if rec.used&pl.mask != 0 {
			return fmt.Errorf("TakePodResources: GPUs of pod %s already in use on %s (score the pod again)", podInfo.Name, pl.node)
		}
		rec.used |= pl.mask
		pl.committed = true
		ns.placed[podInfo.Name] = pl
	}
	if ns.dirty || ns.changed[pl.node] {
		return nil // a re-upload / kgpu_update_node is pending and will carry the mask
	}
	return ns.h.setFreeMask(rec.index, freeOf(rec))
}

func (ns *NvidiaGPUScheduler) TakePodResources(nodeInfo *types.NodeInfo, podInfo *types.PodInfo) error {
	return ns.take(podInfo, false)
}

func (ns *NvidiaGPUScheduler) ReturnPodResources(nodeInfo *types.NodeInfo, podInfo *types.PodInfo) error {
	return ns.take(podInfo, true)
}

func (ns *NvidiaGPUScheduler) GetName() string { return "nvidiagpu" }

// UsingGroupScheduler: false when this plugin fills AllocateFrom itself (default), true in GroupSchedulerMode
// (the reference, gpu_scheduler.go:69-71).
func (ns *NvidiaGPUScheduler) UsingGroupScheduler() bool { return ns.GroupSchedulerMode }
