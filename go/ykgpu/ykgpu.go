// Package ykgpu is the reference-side binding of libykgpu.so: a type that satisfies
// github.com/apache/yunikorn-scheduler-interface/lib/go/api.SchedulerAPI (method set:
// pkg/common/test/schedulerapi_mock.go:88-146) and drives api.ResourceManagerCallback
// (pkg/cache/scheduler_callback.go:42-43), so that pkg/shim is handed this instead of serviceContext.RMProxy
// (pkg/cmd/shim/main.go:56-57) with pkg/shim, pkg/plugin and cache.Context unchanged.
//
// NOT COMPILED IN THIS REPOSITORY: the build image has no Go toolchain and neither the SI nor the Kubernetes modules are
// vendored (SURVEY.md section 0).  The file is complete -- every SchedulerAPI call, the scheduling loop, the snapshot
// builder (strings -> bit sets through the dictionary encoder that ships in the same library), foreign-pod occupancy,
// the slow-path bridge to the unchanged Go PredicateManager and the scheduling-state notifications -- and is written to
// be reviewed next to include/ykgpu.h, include/ykgpu_dict.h and INTEGRATION.md.  Everything with scheduling behaviour
// lives behind the C ABI, where it is tested (tests/ drive the same entry points through ctypes).
//
// Concurrency: one mutex guards the index maps and every cgo call; callbacks into the shim are made WITHOUT it (the
// shim's handlers call back into SchedulerAPI, e.g. task.go:518 releases from inside UpdateAllocation handling).
package ykgpu

/*
#cgo CFLAGS: -I${SRCDIR}/../../include
#cgo LDFLAGS: -L${SRCDIR}/../../yunikorn_k8shim_b200 -lykgpu
#include <stdlib.h>
#include <string.h>
#include "ykgpu.h"
#include "ykgpu_dict.h"

// cgo cannot build arrays of C structs that contain pointers to Go memory: the spec is assembled in C memory
static yk_requirement* yk_go_reqs(uint32_t n) { return (yk_requirement*)calloc(n ? n : 1, sizeof(yk_requirement)); }
static yk_selector_term* yk_go_terms(uint32_t n) { return (yk_selector_term*)calloc(n ? n : 1, sizeof(yk_selector_term)); }
static yk_toleration* yk_go_tols(uint32_t n) { return (yk_toleration*)calloc(n ? n : 1, sizeof(yk_toleration)); }
static yk_taint* yk_go_taints(uint32_t n) { return (yk_taint*)calloc(n ? n : 1, sizeof(yk_taint)); }
static const char** yk_go_strs(uint32_t n) { return (const char**)calloc(n ? n : 1, sizeof(char*)); }
*/
import "C"

import (
	"errors"
	"fmt"
	"math"
	"sort"
	"strconv"
	"strings"
	"sync"
	"time"
	"unsafe"

	"go.yaml.in/yaml/v3"
	v1 "k8s.io/api/core/v1"

	"github.com/apache/yunikorn-scheduler-interface/lib/go/api"
	siCommon "github.com/apache/yunikorn-scheduler-interface/lib/go/common"
	"github.com/apache/yunikorn-scheduler-interface/lib/go/si"
)

// resource dimension order of the engine (yk_config.D = 4): what pkg/common/resource.go puts into si.Resource
var dims = []string{siCommon.CPU, siCommon.Memory, "pods", "ephemeral-storage"}

const none = ^uint32(0)

// ObjectSource is what the adapter reads from the shim's cache to build the bit sets: the pod behind an AllocationKey
// (= pod UID, pkg/common/si_helper.go:75-115) and the node object behind a NodeID.  *external.SchedulerCache satisfies
// it through a two-line wrapper (INTEGRATION.md): GetPod(uid) and GetNode(name).Node().
type ObjectSource interface {
	GetPod(uid string) *v1.Pod
	GetNodeObject(name string) *v1.Node
}

type nodeRec struct {
	name          string
	total         [4]int64
	occupied      [4]int64 // foreign pods (context.go:409-472): part of total the core never sees as available
	schedulable   bool
	present       bool
	rank          uint32
	label, taint  uint64
}

type askRec struct {
	key, app  string
	req       [4]int64
	foreign   bool   // an occupancy record, not a schedulable ask
	node      uint32 // foreign / recovered: the node it sits on
	lastState uint8  // last state reported through UpdateContainerSchedulingState
	prio      int32  // priority and create_seq as first written: every re-push writes them back
	seq       int64
	slow      bool
	exact     bool // slow only for needsGoPredicates: the dictionary encoded the pod's masks exactly (yk_filter_nodes applies)
	present   bool
	ppFlags   C.uint32_t // YK_ASK_NO_PREEMPT_SELF / _OTHER / YK_ASK_ORIGINATOR from the ask's PreemptionPolicy and Originator
	blocked   time.Time  // when the ask was first reported NOFIT / SKIPPED since it last was anything else (zero: not blocked)
	pinNode   uint32     // none, or the node a preemption plan holds for it: written as its required node
	dsNode    string     // a DaemonSet pod's node (CreateTagsForTask's required node), "" otherwise; apart from pinNode
	dsPlanned bool       // yk_preemption_required_node planned it; cleared when it is written again
}

type Engine struct {
	mu    sync.Mutex
	h     *C.yk_engine
	dict  *C.yk_dict
	gen   C.uint64_t // dictionary generation the node / ask bit sets were written under
	cb    api.ResourceManagerCallback
	src   ObjectSource
	rmID  string

	nodeIdx  map[string]uint32
	nodes    []nodeRec
	askIdx   map[string]uint32
	asks     []askRec
	freeAsks []uint32
	appIdx   map[string]uint32
	appName  []string
	appQueue []uint32
	queueIdx map[string]uint32 // "root.a.b" -> index
	queueLeaf []bool
	queueDelay []time.Duration // preemption.delay per queue: how long a blocked ask waits before it may preempt
	nodeSort nodeSort // what yk_node_sort_set last applied: put back when the rest of a configuration is refused
	seq      int64
	stop     chan struct{}
	kick     chan struct{}
}

var _ api.SchedulerAPI = &Engine{}

// New creates the engine.  There is no CPU fallback: without a CUDA device yk_create fails and so does New.
func New(maxNodes, maxAsks, maxApps, maxQueues int, src ObjectSource) (*Engine, error) {
	var cfg C.yk_config
	cfg.abi_version = C.YK_ABI_VERSION
	cfg.D = C.uint32_t(len(dims))
	// the core's default node sort until the configuration arrives (RegisterResourceManager -> applyConfig -> yk_node_sort_set)
	ns := defaultNodeSort()
	cfg.policy, cfg.weights = ns.policy, ns.weights
	cfg.max_nodes, cfg.max_asks, cfg.max_apps, cfg.max_queues = C.uint32_t(maxNodes), C.uint32_t(maxAsks), C.uint32_t(maxApps), C.uint32_t(maxQueues)
	cfg.device = -1
	e := &Engine{src: src, nodeIdx: map[string]uint32{}, askIdx: map[string]uint32{}, appIdx: map[string]uint32{},
		queueIdx: map[string]uint32{}, nodeSort: ns, stop: make(chan struct{}), kick: make(chan struct{}, 1)}
	if rc := C.yk_create(&cfg, &e.h); rc != C.YK_OK {
		return nil, errors.New(C.GoString(C.yk_strerror(rc)))
	}
	e.dict = C.yk_dict_create()
	e.gen = C.yk_dict_generation(e.dict)
	// default tree root -> root.default (deployments/scheduler/yunikorn-configs.yaml:23-32) until the config arrives
	if err := e.setQueues(defaultQueues()); err != nil {
		return nil, err
	}
	return e, nil
}

// SetObjectSource hands over the shim's cache once the shim has built it (the cache does not exist yet when New runs:
// pkg/cmd/shim/main.go creates the SchedulerAPI first, then the shim around it).
func (e *Engine) SetObjectSource(src ObjectSource) {
	e.mu.Lock()
	defer e.mu.Unlock()
	e.src = src
}

func (e *Engine) ck(rc C.int, what string) error {
	if rc == C.YK_OK {
		return nil
	}
	return fmt.Errorf("ykgpu %s: %s (%s)", what, C.GoString(C.yk_strerror(rc)), C.GoString(C.yk_last_error(e.h)))
}

// ---------------------------------------------------------------------------------------------------------------
// queues.yaml (the core's configs.SchedulerConfig, schema evidence: test/e2e/framework/helpers/common/
// test_queues_configs.go:42-60) -> yk_queues_set / yk_queues_priority, and the partition's nodesortpolicy -> yk_node_sort_set
// ---------------------------------------------------------------------------------------------------------------

type queueConf struct {
	Name       string            `yaml:"name"`
	Parent     bool              `yaml:"parent"`
	Resources  struct{ Guaranteed, Max map[string]string } `yaml:"resources"`
	Properties map[string]string `yaml:"properties"`
	Queues     []queueConf       `yaml:"queues"`
}

// the core's configs.NodeSortingPolicy of a partition
type nodeSortConf struct {
	Type            string             `yaml:"type"`
	ResourceWeights map[string]float64 `yaml:"resourceweights"`
}
type schedulerConf struct {
	Partitions []struct {
		Name            string       `yaml:"name"`
		Queues          []queueConf  `yaml:"queues"`
		NodeSortPolicy  nodeSortConf `yaml:"nodesortpolicy"`
	} `yaml:"partitions"`
}

func defaultQueues() []queueConf {
	return []queueConf{{Name: "root", Parent: true, Queues: []queueConf{{Name: "default"}}}}
}

// nodeSort is one yk_node_sort_set setting: YK_POLICY_* and the weights in dims order (the rest of [YK_MAX_D] stays 0)
type nodeSort struct {
	policy  C.uint32_t
	weights [C.YK_MAX_D]C.double
}

// the core's default: fair, vcore = memory = 1 (SURVEY A.3)
func defaultNodeSort() nodeSort {
	s := nodeSort{policy: C.YK_POLICY_FAIR}
	s.weights[0], s.weights[1] = 1, 1
	return s
}

// parseNodeSort maps a partition's nodesortpolicy onto the engine's setting.  type: "" (or no block) = fair; "fair" and
// "binpacking" are exact names; anything else is an error.  resourceweights: absent = the core default; a weight on a
// resource outside dims (e.g. nvidia.com/gpu) cannot be honoured -- the engine does not track that resource -- so it refuses
// the configuration rather than sort by something else.
func parseNodeSort(c nodeSortConf) (nodeSort, error) {
	s := defaultNodeSort()
	switch c.Type {
	case "", "fair":
	case "binpacking":
		s.policy = C.YK_POLICY_BINPACKING
	default:
		return s, fmt.Errorf("ykgpu: nodesortpolicy type %q: not fair or binpacking", c.Type)
	}
	if len(c.ResourceWeights) == 0 {
		return s, nil
	}
	s.weights = [C.YK_MAX_D]C.double{}
	for name, w := range c.ResourceWeights {
		k := -1
		for i, d := range dims {
			if d == name {
				k = i
			}
		}
		if k < 0 {
			return s, fmt.Errorf("ykgpu: nodesortpolicy resourceweights: resource %q is not one the engine sorts by (%s)", name,
				strings.Join(dims, ", "))
		}
		if math.IsNaN(w) || math.IsInf(w, 0) {
			return s, fmt.Errorf("ykgpu: nodesortpolicy resourceweights: weight of %q is not a finite number", name)
		}
		s.weights[k] = C.double(w)
	}
	return s, nil
}

// setNodeSort: yk_node_sort_set refuses (and keeps the old setting) when a present node would score NaN under the new one
func (e *Engine) setNodeSort(s nodeSort) error {
	if err := e.ck(C.yk_node_sort_set(e.h, s.policy, &s.weights[0]), "yk_node_sort_set"); err != nil {
		return err
	}
	e.nodeSort = s
	return nil
}

// quantity: the core's resources.NewResourceFromConf -- plain integers, "vcore" in milli units when suffixed with m,
// memory with the binary / decimal suffixes of resource.Quantity.  The library parses Kubernetes quantities
// (include/ykgpu_pod.h yk_quantity_value); the configuration only uses the subset below.
func quantity(name, s string) int64 {
	s = strings.TrimSpace(s)
	mult := int64(1)
	for suf, m := range map[string]int64{"Ki": 1 << 10, "Mi": 1 << 20, "Gi": 1 << 30, "Ti": 1 << 40, "k": 1e3, "M": 1e6, "G": 1e9, "T": 1e12} {
		if strings.HasSuffix(s, suf) {
			s, mult = strings.TrimSuffix(s, suf), m
			break
		}
	}
	if name == siCommon.CPU {
		if strings.HasSuffix(s, "m") {
			v, _ := strconv.ParseInt(strings.TrimSuffix(s, "m"), 10, 64)
			return v
		}
		v, _ := strconv.ParseInt(s, 10, 64)
		return v * 1000
	}
	v, _ := strconv.ParseInt(s, 10, 64)
	return v * mult
}

func resVec(m map[string]string) [4]int64 {
	v := [4]int64{-1, -1, -1, -1} // -1 = not set
	for k, name := range dims {
		if s, ok := m[name]; ok {
			v[k] = quantity(name, s)
		}
	}
	return v
}

func (e *Engine) setQueues(root []queueConf) error {
	var parent []C.uint32_t
	var guar, max [][4]int64
	var sortPol []C.uint8_t
	var off []C.int32_t
	var fence, ppFence []C.uint8_t
	var delay []time.Duration
	idx := map[string]uint32{}
	var leaf []bool
	var walk func(q queueConf, p uint32, path string)
	walk = func(q queueConf, p uint32, path string) {
		me := uint32(len(parent))
		parent = append(parent, C.uint32_t(p))
		guar, max = append(guar, resVec(q.Resources.Guaranteed)), append(max, resVec(q.Resources.Max))
		s := C.uint8_t(C.YK_SORT_FIFO)
		if q.Properties["application.sort.policy"] == "fair" {
			s = C.YK_SORT_FAIR
		}
		sortPol = append(sortPol, s)
		o, _ := strconv.ParseInt(q.Properties["priority.offset"], 10, 32)
		off = append(off, C.int32_t(o))
		f := C.uint8_t(0)
		if q.Properties["priority.policy"] == "fence" {
			f = 1
		}
		fence = append(fence, f)
		pf := C.uint8_t(0)
		if q.Properties["preemption.policy"] == "fence" {
			pf = 1
		}
		ppFence = append(ppFence, pf)
		d, err := time.ParseDuration(q.Properties["preemption.delay"])
		if err != nil || d <= 0 {
			d = 30 * time.Second // the core's default
		}
		delay = append(delay, d)
		idx[path] = me
		leaf = append(leaf, len(q.Queues) == 0 && !q.Parent)
		for _, c := range q.Queues {
			walk(c, me, path+"."+c.Name)
		}
	}
	for _, q := range root {
		walk(q, none, q.Name)
	}
	n := len(parent)
	g, m := make([]C.int64_t, 4*n), make([]C.int64_t, 4*n) // [D][q] column-major
	for i := 0; i < n; i++ {
		for k := 0; k < 4; k++ {
			g[k*n+i], m[k*n+i] = C.int64_t(guar[i][k]), C.int64_t(max[i][k])
		}
	}
	// allocated == NULL: the library sums what the present applications hold up the new tree (yk_queues_set)
	if err := e.ck(C.yk_queues_set(e.h, C.uint32_t(n), &parent[0], &g[0], &m[0], nil, &sortPol[0]), "yk_queues_set"); err != nil {
		return err
	}
	if err := e.ck(C.yk_queues_priority(e.h, C.uint32_t(n), &off[0], &fence[0]), "yk_queues_priority"); err != nil {
		return err
	}
	if err := e.ck(C.yk_queues_preemption(e.h, C.uint32_t(n), &ppFence[0]), "yk_queues_preemption"); err != nil {
		return err
	}
	e.queueIdx, e.queueLeaf, e.queueDelay = idx, leaf, delay
	return nil
}

func (e *Engine) applyConfig(cfg string) error {
	if strings.TrimSpace(cfg) == "" {
		return nil
	}
	var sc schedulerConf
	if err := yaml.Unmarshal([]byte(cfg), &sc); err != nil {
		return err
	}
	if len(sc.Partitions) == 0 {
		return nil
	}
	// one engine = one partition (a second partition is a second Engine on another GPU: DESIGN.md "multi-GPU")
	p := sc.Partitions[0]
	// all or nothing: everything is parsed and validated before the engine changes; the node sort goes first and is put back
	// when the queue tree is refused, so the shim's old configuration stays in force either way
	ns, err := parseNodeSort(p.NodeSortPolicy)
	if err != nil {
		return err
	}
	prev := e.nodeSort
	if err := e.setNodeSort(ns); err != nil {
		return err
	}
	if err := e.setQueues(p.Queues); err != nil {
		// the node tables are those the first call saw (e.mu is held throughout): this fails only where prev already made the
		// cycles fail (a node scoring NaN), and the error then says so
		if rerr := e.setNodeSort(prev); rerr != nil {
			return fmt.Errorf("%v; putting the previous node sort back: %v", err, rerr)
		}
		return err
	}
	return nil
}

// RegisterResourceManager: pkg/shim/scheduler.go:147-167 hands over the callback object and the queues.yaml text
func (e *Engine) RegisterResourceManager(req *si.RegisterResourceManagerRequest, cb api.ResourceManagerCallback) (*si.RegisterResourceManagerResponse, error) {
	e.mu.Lock()
	defer e.mu.Unlock()
	e.cb, e.rmID = cb, req.RmID
	if err := e.applyConfig(req.Config); err != nil {
		return nil, err
	}
	go e.loop()
	return &si.RegisterResourceManagerResponse{}, nil
}

// UpdateConfiguration: a changed queues.yaml.  yk_queues_set refuses a tree that drops a queue applications still sit
// in (YK_ERR_STATE), parseNodeSort an unknown policy or a weight on an untracked resource, yk_node_sort_set a setting under
// which a node scores NaN: the error goes back to the shim, which keeps the old configuration (as the core does), and so does
// the engine.  A new nodesortpolicy orders the nodes from the next cycle on.
func (e *Engine) UpdateConfiguration(req *si.UpdateConfigurationRequest) error {
	e.mu.Lock()
	defer e.mu.Unlock()
	return e.applyConfig(req.Config)
}

// ---------------------------------------------------------------------------------------------------------------
// nodes
// ---------------------------------------------------------------------------------------------------------------

func vec(r *si.Resource) [4]int64 {
	var v [4]int64
	if r != nil {
		for k, name := range dims {
			if q, ok := r.Resources[name]; ok {
				v[k] = q.Value
			}
		}
	}
	return v
}

// nodeBits: labels / taints / spec.unschedulable of the node object -> the dictionary's bit sets
func (e *Engine) nodeBits(idx uint32, name string) (label, taint uint64) {
	var obj *v1.Node
	if e.src != nil {
		obj = e.src.GetNodeObject(name)
	}
	cName := C.CString(name)
	defer C.free(unsafe.Pointer(cName))
	var keys, vals **C.char
	var taints *C.yk_taint
	nl, nt := 0, 0
	unsched := C.int32_t(0)
	var held []unsafe.Pointer
	hold := func(s string) *C.char { p := C.CString(s); held = append(held, unsafe.Pointer(p)); return p }
	defer func() {
		for _, p := range held {
			C.free(p)
		}
	}()
	if obj != nil {
		nl = len(obj.Labels)
		keys, vals = C.yk_go_strs(C.uint32_t(nl)), C.yk_go_strs(C.uint32_t(nl))
		defer C.free(unsafe.Pointer(keys))
		defer C.free(unsafe.Pointer(vals))
		ks := unsafe.Slice(keys, nl+1)
		vs := unsafe.Slice(vals, nl+1)
		i := 0
		for k, v := range obj.Labels {
			ks[i], vs[i] = hold(k), hold(v)
			i++
		}
		nt = len(obj.Spec.Taints)
		taints = C.yk_go_taints(C.uint32_t(nt))
		defer C.free(unsafe.Pointer(taints))
		ts := unsafe.Slice(taints, nt+1)
		for i, t := range obj.Spec.Taints {
			ts[i].key, ts[i].value, ts[i].effect = hold(t.Key), hold(t.Value), effectOf(t.Effect)
		}
		if obj.Spec.Unschedulable {
			unsched = 1
		}
	}
	var lb, tb C.uint64_t
	C.yk_dict_node(e.dict, C.uint32_t(idx), cName, C.uint32_t(nl), keys, vals, C.uint32_t(nt), taints, unsched, &lb, &tb)
	return uint64(lb), uint64(tb)
}

func effectOf(ef v1.TaintEffect) C.uint32_t {
	switch ef {
	case v1.TaintEffectNoSchedule:
		return C.YK_EFFECT_NO_SCHEDULE
	case v1.TaintEffectPreferNoSchedule:
		return C.YK_EFFECT_PREFER_NO_SCHEDULE
	case v1.TaintEffectNoExecute:
		return C.YK_EFFECT_NO_EXECUTE
	}
	return C.YK_EFFECT_ALL
}

// pushNode writes one node to the engine.  avail = total - occupied - (what the engine itself has allocated there):
// the engine's current availability moves by the change of (total - occupied), it is never reset to total.
func (e *Engine) pushNode(idx uint32, n *nodeRec, availDelta [4]int64, isNew bool) error {
	i := C.uint32_t(idx)
	var total, avail [4]C.int64_t
	if isNew {
		for k := 0; k < 4; k++ {
			total[k], avail[k] = C.int64_t(n.total[k]), C.int64_t(n.total[k]-n.occupied[k])
		}
	} else {
		var cur [4]C.int64_t
		if err := e.ck(C.yk_nodes_available(e.h, 1, &i, &cur[0]), "yk_nodes_available"); err != nil {
			return err
		}
		for k := 0; k < 4; k++ {
			total[k], avail[k] = C.int64_t(n.total[k]), cur[k]+C.int64_t(availDelta[k])
		}
	}
	flags := C.uint32_t(0)
	if n.schedulable {
		flags = C.YK_NODE_SCHEDULABLE
	}
	taint, label, rank := C.uint64_t(n.taint), C.uint64_t(n.label), C.uint32_t(n.rank)
	return e.ck(C.yk_nodes_upsert(e.h, 1, &i, &total[0], &avail[0], &taint, &label, &rank, &flags), "yk_nodes_upsert")
}

// refreshRanks: name_rank must preserve the Go string order of the NodeIDs (tie-break of the node iterator, SURVEY
// A.3).  Ranks are re-dealt with gaps when a new name does not fit between its neighbours; only nodes whose rank
// changed are written again.
func (e *Engine) refreshRanks() error {
	order := make([]int, 0, len(e.nodes))
	for i := range e.nodes {
		if e.nodes[i].present {
			order = append(order, i)
		}
	}
	sort.Slice(order, func(a, b int) bool { return e.nodes[order[a]].name < e.nodes[order[b]].name })
	for pos, i := range order {
		want := uint32(pos+1) << 8 // room for 255 insertions between neighbours before the next full re-deal
		n := &e.nodes[i]
		lo, hi := uint32(0), ^uint32(0)
		if pos > 0 {
			lo = e.nodes[order[pos-1]].rank
		}
		if pos+1 < len(order) && e.nodes[order[pos+1]].rank != 0 {
			hi = e.nodes[order[pos+1]].rank
		}
		if n.rank > lo && n.rank < hi && n.rank != 0 {
			continue // still in order: keep
		}
		if lo+1 < hi && n.rank == 0 && hi != ^uint32(0) {
			want = lo + (hi-lo)/2
		}
		n.rank = want
		if err := e.pushNode(uint32(i), n, [4]int64{}, false); err != nil {
			return err
		}
	}
	return nil
}

// UpdateNode: call sites pkg/cache/context.go:256 (drain), :1610,:1630,:1635 (register / update), :1656 (remove)
func (e *Engine) UpdateNode(req *si.NodeRequest) error {
	e.mu.Lock()
	accepted := make([]*si.AcceptedNode, 0, len(req.Nodes))
	rejected := make([]*si.RejectedNode, 0)
	needRanks := false
	for _, n := range req.Nodes {
		idx, known := e.nodeIdx[n.NodeID]
		switch n.Action {
		case si.NodeInfo_DECOMISSION:
			if known {
				i := C.uint32_t(idx)
				C.yk_nodes_remove(e.h, 1, &i)
				C.yk_dict_node_remove(e.dict, i)
				e.nodes[idx].present = false
				delete(e.nodeIdx, n.NodeID)
			}
			continue
		case si.NodeInfo_DRAIN_NODE, si.NodeInfo_DRAIN_TO_SCHEDULABLE:
			// cordon / uncordon carry no resources (context.go:247-257): a flag-only update
			if !known {
				rejected = append(rejected, &si.RejectedNode{NodeID: n.NodeID, Reason: "unknown node"})
				continue
			}
			rec := &e.nodes[idx]
			rec.schedulable = n.Action == si.NodeInfo_DRAIN_TO_SCHEDULABLE
			rec.label, rec.taint = e.nodeBits(idx, rec.name) // spec.unschedulable is a taint bit as well
			if err := e.pushNode(idx, rec, [4]int64{}, false); err != nil {
				rejected = append(rejected, &si.RejectedNode{NodeID: n.NodeID, Reason: err.Error()})
			}
			continue
		}
		// CREATE, CREATE_DRAIN, UPDATE
		isNew := !known
		if isNew {
			idx = uint32(len(e.nodes))
			for i := range e.nodes { // reuse the slot of a removed node
				if !e.nodes[i].present {
					idx = uint32(i)
					break
				}
			}
			if int(idx) == len(e.nodes) {
				e.nodes = append(e.nodes, nodeRec{})
			}
			e.nodes[idx] = nodeRec{name: n.NodeID, present: true, schedulable: n.Action != si.NodeInfo_CREATE_DRAIN}
			e.nodeIdx[n.NodeID] = idx
			needRanks = true
		}
		rec := &e.nodes[idx]
		newTotal := vec(n.SchedulableResource)
		var delta [4]int64
		for k := 0; k < 4; k++ {
			delta[k] = newTotal[k] - rec.total[k] // capacity change moves availability by the same amount
		}
		rec.total = newTotal
		rec.label, rec.taint = e.nodeBits(idx, rec.name)
		if err := e.pushNode(idx, rec, delta, isNew); err != nil {
			rejected = append(rejected, &si.RejectedNode{NodeID: n.NodeID, Reason: err.Error()})
			continue
		}
		accepted = append(accepted, &si.AcceptedNode{NodeID: n.NodeID})
	}
	var err error
	if needRanks {
		err = e.refreshRanks()
	}
	cb := e.cb
	e.mu.Unlock()
	// Accepted / Rejected must come from another goroutine: registerNodes waits on a WaitGroup (context.go:1580-1623)
	if cb != nil && (len(accepted) > 0 || len(rejected) > 0) {
		go cb.UpdateNode(&si.NodeResponse{Accepted: accepted, Rejected: rejected}) //nolint:errcheck
	}
	e.wake()
	return err
}

// ---------------------------------------------------------------------------------------------------------------
// applications
// ---------------------------------------------------------------------------------------------------------------

// UpdateApplication: pkg/cache/application.go:423 (New, with the Ugi the shim resolved, :430) and :597 (Remove)
func (e *Engine) UpdateApplication(req *si.ApplicationRequest) error {
	e.mu.Lock()
	acc := make([]*si.AcceptedApplication, 0, len(req.New))
	rej := make([]*si.RejectedApplication, 0)
	for _, a := range req.New {
		q, ok := e.queueIdx[a.QueueName]
		if !ok || !e.queueLeaf[q] {
			// the core's placement rules would create / pick a queue; this adapter takes the queue the shim names
			rej = append(rej, &si.RejectedApplication{ApplicationID: a.ApplicationID, Reason: "queue " + a.QueueName + " is not a leaf of the configured tree"})
			continue
		}
		idx, known := e.appIdx[a.ApplicationID]
		if !known {
			idx = uint32(len(e.appName))
			e.appName = append(e.appName, a.ApplicationID)
			e.appQueue = append(e.appQueue, q)
			e.appIdx[a.ApplicationID] = idx
		}
		i, cq, t := C.uint32_t(idx), C.uint32_t(q), C.int64_t(time.Now().UnixNano()) // submission time: unique (SURVEY A.6)
		if err := e.ck(C.yk_apps_upsert(e.h, 1, &i, &cq, &t), "yk_apps_upsert"); err != nil {
			rej = append(rej, &si.RejectedApplication{ApplicationID: a.ApplicationID, Reason: err.Error()})
			continue
		}
		acc = append(acc, &si.AcceptedApplication{ApplicationID: a.ApplicationID})
	}
	for _, r := range req.Remove {
		if idx, ok := e.appIdx[r.ApplicationID]; ok {
			i := C.uint32_t(idx)
			C.yk_apps_remove(e.h, 1, &i)
			delete(e.appIdx, r.ApplicationID)
		}
	}
	cb := e.cb
	e.mu.Unlock()
	if cb != nil && (len(acc) > 0 || len(rej) > 0) {
		go cb.UpdateApplication(&si.ApplicationResponse{Accepted: acc, Rejected: rej}) //nolint:errcheck
	}
	return nil
}

// ---------------------------------------------------------------------------------------------------------------
// asks, allocations, releases
// ---------------------------------------------------------------------------------------------------------------

// needsGoPredicates: what does not reduce to the bit sets (SURVEY A.4) stays with the unchanged PredicateManager
func needsGoPredicates(p *v1.Pod) bool {
	if p == nil {
		return true // nothing known about the pod: let the Go path decide
	}
	for _, c := range p.Spec.Containers {
		for _, port := range c.Ports {
			if port.HostPort != 0 {
				return true
			}
		}
	}
	for _, v := range p.Spec.Volumes {
		if v.PersistentVolumeClaim != nil || v.Ephemeral != nil {
			return true
		}
	}
	if a := p.Spec.Affinity; a != nil && (a.PodAffinity != nil || a.PodAntiAffinity != nil) {
		return true
	}
	return len(p.Spec.TopologySpreadConstraints) > 0
}

// daemonSetNode: the required node of a DaemonSet pod as the shim's CreateTagsForTask finds it (pkg/common/si_helper.go:33-58):
// for an owner of kind DaemonSet, the last metadata.name match field of its required node affinity, first value; "" when
// there is none
func daemonSetNode(p *v1.Pod) string {
	node := ""
	for _, o := range p.GetOwnerReferences() {
		if o.Kind != "DaemonSet" {
			continue
		}
		a := p.Spec.Affinity
		if a == nil || a.NodeAffinity == nil || a.NodeAffinity.RequiredDuringSchedulingIgnoredDuringExecution == nil {
			continue
		}
		for _, t := range a.NodeAffinity.RequiredDuringSchedulingIgnoredDuringExecution.NodeSelectorTerms {
			for _, m := range t.MatchFields {
				if m.Key == "metadata.name" && len(m.Values) > 0 {
					node = m.Values[0]
				}
			}
		}
	}
	return node
}

// podMasks: nodeSelector + required node affinity + tolerations + spec.nodeName -> yk_pod_masks.  exact: the dictionary
// encoded all of them (it did not set YK_ASK_SLOWPATH itself; needsGoPredicates may still have).  A DaemonSet pod is encoded
// against its node (yk_dict_pod_required_node), which also becomes its required node; dsNode names it.
func (e *Engine) podMasks(p *v1.Pod) (out C.yk_pod_masks, exact bool, dsNode string) {
	out.required_node = C.YK_NONE
	if p == nil {
		out.flags = C.YK_ASK_SLOWPATH
		return out, false, ""
	}
	var held []unsafe.Pointer
	hold := func(s string) *C.char { c := C.CString(s); held = append(held, unsafe.Pointer(c)); return c }
	keep := func(p unsafe.Pointer) { held = append(held, p) }
	defer func() {
		for _, x := range held {
			C.free(x)
		}
	}()
	var spec C.yk_pod_spec
	ns := len(p.Spec.NodeSelector)
	sk, sv := C.yk_go_strs(C.uint32_t(ns)), C.yk_go_strs(C.uint32_t(ns))
	keep(unsafe.Pointer(sk))
	keep(unsafe.Pointer(sv))
	i := 0
	for k, v := range p.Spec.NodeSelector {
		unsafe.Slice(sk, ns+1)[i], unsafe.Slice(sv, ns+1)[i] = hold(k), hold(v)
		i++
	}
	spec.n_selector, spec.selector_keys, spec.selector_values = C.uint32_t(ns), sk, sv
	reqs := func(in []v1.NodeSelectorRequirement) (*C.yk_requirement, C.uint32_t) {
		r := C.yk_go_reqs(C.uint32_t(len(in)))
		keep(unsafe.Pointer(r))
		rs := unsafe.Slice(r, len(in)+1)
		for i, x := range in {
			vals := C.yk_go_strs(C.uint32_t(len(x.Values)))
			keep(unsafe.Pointer(vals))
			for j, v := range x.Values {
				unsafe.Slice(vals, len(x.Values)+1)[j] = hold(v)
			}
			rs[i].key, rs[i].n_values, rs[i].values = hold(x.Key), C.uint32_t(len(x.Values)), vals
			switch x.Operator {
			case v1.NodeSelectorOpIn:
				rs[i].op = C.YK_OP_IN
			case v1.NodeSelectorOpNotIn:
				rs[i].op = C.YK_OP_NOT_IN
			case v1.NodeSelectorOpExists:
				rs[i].op = C.YK_OP_EXISTS
			case v1.NodeSelectorOpDoesNotExist:
				rs[i].op = C.YK_OP_DOES_NOT_EXIST
			case v1.NodeSelectorOpGt:
				rs[i].op = C.YK_OP_GT
			case v1.NodeSelectorOpLt:
				rs[i].op = C.YK_OP_LT
			}
		}
		return r, C.uint32_t(len(in))
	}
	if a := p.Spec.Affinity; a != nil && a.NodeAffinity != nil && a.NodeAffinity.RequiredDuringSchedulingIgnoredDuringExecution != nil {
		spec.has_required_affinity = 1
		in := a.NodeAffinity.RequiredDuringSchedulingIgnoredDuringExecution.NodeSelectorTerms
		terms := C.yk_go_terms(C.uint32_t(len(in)))
		keep(unsafe.Pointer(terms))
		for i, t := range in {
			ts := unsafe.Slice(terms, len(in)+1)
			ts[i].expressions, ts[i].n_expressions = reqs(t.MatchExpressions)
			ts[i].fields, ts[i].n_fields = reqs(t.MatchFields)
		}
		spec.n_terms, spec.terms = C.uint32_t(len(in)), terms
	}
	tols := C.yk_go_tols(C.uint32_t(len(p.Spec.Tolerations)))
	keep(unsafe.Pointer(tols))
	for i, t := range p.Spec.Tolerations {
		ts := unsafe.Slice(tols, len(p.Spec.Tolerations)+1)
		ts[i].key, ts[i].value, ts[i].effect = hold(t.Key), hold(t.Value), effectOf(t.Effect)
		if t.Operator == v1.TolerationOpExists {
			ts[i].op = C.YK_TOL_EXISTS
		}
	}
	spec.n_tolerations, spec.tolerations = C.uint32_t(len(p.Spec.Tolerations)), tols
	if p.Spec.NodeName != "" {
		spec.node_name = hold(p.Spec.NodeName)
	}
	if dsNode = daemonSetNode(p); dsNode != "" {
		C.yk_dict_pod_required_node(e.dict, &spec, hold(dsNode), &out)
	} else {
		C.yk_dict_pod(e.dict, &spec, &out)
	}
	exact = out.flags&C.YK_ASK_SLOWPATH == 0
	if needsGoPredicates(p) {
		out.flags |= C.YK_ASK_SLOWPATH
	}
	return out, exact, dsNode
}

// dictionary handed out new bits while compiling a pod: node bit sets (and key-only tolerations) were extended
func (e *Engine) syncDictionary() error {
	g := C.yk_dict_generation(e.dict)
	if g == e.gen {
		return nil
	}
	e.gen = g
	for i := range e.nodes {
		n := &e.nodes[i]
		if !n.present {
			continue
		}
		var lb, tb C.uint64_t
		C.yk_dict_node_bits(e.dict, C.uint32_t(i), &lb, &tb)
		if uint64(lb) != n.label || uint64(tb) != n.taint {
			n.label, n.taint = uint64(lb), uint64(tb)
			if err := e.pushNode(uint32(i), n, [4]int64{}, false); err != nil {
				return err
			}
		}
	}
	// pending asks whose tolerations name a key that just got a bit are re-encoded (cheap: only pending, only on growth)
	for i := range e.asks {
		a := &e.asks[i]
		if a.present && !a.foreign && a.lastState != C.YK_ST_ALLOCATED {
			if err := e.pushAsk(uint32(i), a, nil); err != nil {
				return err
			}
		}
	}
	return nil
}

func (e *Engine) newAskSlot() uint32 {
	if n := len(e.freeAsks); n > 0 {
		idx := e.freeAsks[n-1]
		e.freeAsks = e.freeAsks[:n-1]
		return idx
	}
	e.asks = append(e.asks, askRec{})
	return uint32(len(e.asks) - 1)
}

// pushAsk (re)writes a pending ask; alloc != nil on the first write, which fixes its priority and create_seq (creation time)
func (e *Engine) pushAsk(idx uint32, a *askRec, alloc *si.Allocation) error {
	var pod *v1.Pod
	if e.src != nil {
		pod = e.src.GetPod(a.key)
	}
	m, exact, dsNode := e.podMasks(pod)
	a.slow = m.flags&C.YK_ASK_SLOWPATH != 0
	a.exact = exact
	a.dsNode, a.dsPlanned = dsNode, false // a write clears the engine's plan
	app, ok := e.appIdx[a.app]
	if !ok {
		return fmt.Errorf("ask %s: unknown application %s", a.key, a.app)
	}
	var rq [4]C.int64_t
	for k := 0; k < 4; k++ {
		rq[k] = C.int64_t(a.req[k])
	}
	if alloc != nil {
		created, _ := strconv.ParseInt(alloc.AllocationTags[siCommon.CreationTime], 10, 64)
		e.seq++
		a.prio, a.seq = alloc.Priority, created<<20|e.seq&0xFFFFF // seconds tie: break by arrival (SURVEY A.6)
		a.lastState = C.YK_ST_PENDING
		a.ppFlags, a.pinNode = 0, none
		if pp := alloc.PreemptionPolicy; pp != nil {
			if !pp.AllowPreemptSelf {
				a.ppFlags |= C.YK_ASK_NO_PREEMPT_SELF
			}
			if !pp.AllowPreemptOther {
				a.ppFlags |= C.YK_ASK_NO_PREEMPT_OTHER
			}
		}
		if alloc.Originator {
			a.ppFlags |= C.YK_ASK_ORIGINATOR
		}
	}
	prio, seq := C.int32_t(a.prio), C.int64_t(a.seq)
	i, capp := C.uint32_t(idx), C.uint32_t(app)
	tol, need, deny, rn, fl := m.tolerated_bits, m.required_bits, m.forbidden_bits, m.required_node, m.flags|a.ppFlags
	if a.pinNode != none {
		rn = C.uint32_t(a.pinNode)
	}
	return e.ck(C.yk_asks_upsert(e.h, 1, &i, &rq[0], &tol, &need, &deny, &prio, &seq, &capp, &rn, &fl, nil), "yk_asks_upsert")
}

// occupy: a pod that holds resources on a node without being scheduled by this engine -- a foreign pod
// (context.go:409-472, tagged siCommon.Foreign) or a YuniKorn pod found bound on recovery: the node's occupancy grows by
// d (its request when it arrives, the change of its request on a resize, minus its request on the release) and its
// availability drops by d, in one node push.
func (e *Engine) occupy(node uint32, d [4]int64) error {
	n := &e.nodes[node]
	var delta [4]int64
	for k := 0; k < 4; k++ {
		n.occupied[k] += d[k]
		delta[k] = -d[k]
	}
	return e.pushNode(node, n, delta, false)
}

func neg(v [4]int64) [4]int64 {
	for k := range v {
		v[k] = -v[k]
	}
	return v
}

// resize follows an in-place pod resize (KEP-1287): the shim re-sends an allocation under a known key whenever
// common.GetPodResource of the pod changes (Task.SetTaskPod, task.go:633-647; foreign pods, context.go:427-433).  An
// unchanged vector is ignored.  A YuniKorn ask, pending or bound, takes the new request in the engine (yk_asks_resize:
// the bound node, the queues, the application and the user limits follow); a foreign or recovered allocation moves its
// node's occupancy by the change.
func (e *Engine) resize(idx uint32, req [4]int64) error {
	a := &e.asks[idx]
	if req == a.req {
		return nil
	}
	if a.foreign {
		var d [4]int64
		for k := 0; k < 4; k++ {
			d[k] = req[k] - a.req[k]
		}
		a.req = req
		return e.occupy(a.node, d)
	}
	var rq [4]C.int64_t
	for k := 0; k < 4; k++ {
		rq[k] = C.int64_t(req[k])
	}
	i := C.uint32_t(idx)
	if err := e.ck(C.yk_asks_resize(e.h, 1, &i, &rq[0]), "yk_asks_resize"); err != nil {
		return err
	}
	a.req = req
	a.dsPlanned = false // a resize clears the engine's plan
	return nil
}

// UpdateAllocation: asks are si.Allocation without NodeID (si_helper.go:75-115, sent from task.go:311-334); with a
// NodeID they are existing / foreign allocations; releases come from task.go:518 and context.go:459
func (e *Engine) UpdateAllocation(req *si.AllocationRequest) error {
	e.mu.Lock()
	defer e.mu.Unlock()
	var firstErr error
	note := func(err error) {
		if err != nil && firstErr == nil {
			firstErr = err
		}
	}
	for _, al := range req.Allocations {
		if idx, known := e.askIdx[al.AllocationKey]; known {
			note(e.resize(idx, vec(al.ResourcePerAlloc)))
			continue
		}
		rec := askRec{key: al.AllocationKey, app: al.ApplicationID, req: vec(al.ResourcePerAlloc), present: true}
		if al.NodeID != "" {
			nidx, ok := e.nodeIdx[al.NodeID]
			if !ok {
				note(fmt.Errorf("allocation %s on unknown node %s", al.AllocationKey, al.NodeID))
				continue
			}
			rec.foreign, rec.node = true, nidx
			idx := e.newAskSlot()
			e.asks[idx] = rec
			e.askIdx[al.AllocationKey] = idx
			note(e.occupy(nidx, rec.req))
			continue
		}
		idx := e.newAskSlot()
		e.asks[idx] = rec
		e.askIdx[al.AllocationKey] = idx
		note(e.pushAsk(idx, &e.asks[idx], al))
	}
	note(e.syncDictionary())
	if req.Releases != nil {
		for _, r := range req.Releases.AllocationsToRelease {
			idx, ok := e.askIdx[r.AllocationKey]
			if !ok {
				continue
			}
			a := &e.asks[idx]
			switch {
			case a.foreign:
				note(e.occupy(a.node, neg(a.req)))
			case a.lastState == C.YK_ST_ALLOCATED:
				i := C.uint32_t(idx)
				note(e.ck(C.yk_release(e.h, 1, &i), "yk_release"))
			default:
				i := C.uint32_t(idx)
				note(e.ck(C.yk_asks_remove(e.h, 1, &i), "yk_asks_remove"))
			}
			a.present = false
			delete(e.askIdx, r.AllocationKey)
			e.freeAsks = append(e.freeAsks, idx)
		}
	}
	e.wake()
	return firstErr
}

// ---------------------------------------------------------------------------------------------------------------
// the scheduling goroutine
// ---------------------------------------------------------------------------------------------------------------

func (e *Engine) wake() {
	select {
	case e.kick <- struct{}{}:
	default:
	}
}

func (e *Engine) Stop() {
	close(e.stop)
	e.mu.Lock()
	defer e.mu.Unlock()
	C.yk_destroy(e.h)
	C.yk_dict_destroy(e.dict)
}

// loop: one yk_cycle per wake-up; what it returns is handed to the shim exactly as the core's
// notifyRMNewAllocation / UpdateContainerSchedulingState do (scheduler_callback.go:49-91, :218-222 consume them).
func (e *Engine) loop() {
	out := make([]C.yk_binding, 1<<16)
	slow := make([]C.uint32_t, 1<<12)
	for {
		select {
		case <-e.stop:
			return
		case <-e.kick:
		case <-time.After(100 * time.Millisecond): // asks that failed are tried again (node changes arrive as kicks)
		}
		e.mu.Lock()
		var n, nslow C.uint32_t
		rc := C.yk_cycle(e.h, C.uint32_t(len(out)), &out[0], &n, &slow[0], C.uint32_t(len(slow)), &nslow)
		resp := &si.AllocationResponse{}
		// a cycle that broke off still returns the bindings it made: they are real, hand them over
		for i := 0; i < int(n); i++ {
			a, node := uint32(out[i].ask), uint32(out[i].node)
			rec := &e.asks[a]
			rec.lastState = C.YK_ST_ALLOCATED
			resp.New = append(resp.New, &si.Allocation{AllocationKey: rec.key, ApplicationID: rec.app, NodeID: e.nodes[node].name,
				ResourcePerAlloc: nil /* the shim only reads key, application and node: scheduler_callback.go:53-76 */})
		}
		var states []*si.UpdateContainerSchedulingStateRequest
		var preempted *si.AllocationResponse
		if rc == C.YK_OK {
			states = e.collectStates()
			preempted = e.preempt()
			if ds := e.preemptDaemons(); ds != nil {
				if preempted == nil {
					preempted = ds
				} else {
					preempted.Released = append(preempted.Released, ds.Released...)
				}
			}
		}
		slowKeys := make([]uint32, 0, int(nslow))
		for i := 0; i < int(nslow); i++ {
			slowKeys = append(slowKeys, uint32(slow[i]))
		}
		cb := e.cb
		e.mu.Unlock()
		if rc != C.YK_OK {
			// the error text is in yk_last_error; the loop goes on with the next kick
			_ = rc
		}
		if cb == nil {
			continue
		}
		if len(resp.New) > 0 {
			_ = cb.UpdateAllocation(resp) // -> AssumePod + bind, one pod at a time (scheduler_callback.go:53-91, task.go:348)
		}
		for _, s := range states {
			cb.UpdateContainerSchedulingState(s)
		}
		if preempted != nil {
			_ = cb.UpdateAllocation(preempted) // -> ForgetPod + the task's release event (scheduler_callback.go:102-115)
		}
		e.slowPath(cb, slowKeys)
	}
}

// preempt: the core's preemption for queues below their guarantee, once per loop, for the asks blocked (NOFIT / SKIPPED)
// for at least their queue's preemption.delay, oldest first (yk_preemption_plan, DESIGN.md §2 item 9).  A plan's victims are
// released here and handed to the shim as preempted; the preemptor is pinned to the planned node through its required node,
// so the next cycle places it there.  Called with e.mu held; nil when nothing was preempted.
func (e *Engine) preempt() *si.AllocationResponse {
	now := time.Now()
	var asks []C.uint32_t
	for i := range e.asks {
		a := &e.asks[i]
		if !a.present || a.foreign || a.slow || a.blocked.IsZero() || a.pinNode != none || a.dsNode != "" {
			continue
		}
		d := 30 * time.Second
		if q := e.appQueue[e.appIdx[a.app]]; int(q) < len(e.queueDelay) {
			d = e.queueDelay[q]
		}
		if now.Sub(a.blocked) >= d {
			asks = append(asks, C.uint32_t(i))
		}
	}
	if len(asks) == 0 {
		return nil
	}
	sort.Slice(asks, func(x, y int) bool { return e.asks[asks[x]].blocked.Before(e.asks[asks[y]].blocked) })
	n := len(asks)
	status, node := make([]C.uint32_t, n), make([]C.uint32_t, n)
	off, victims := make([]C.uint32_t, n+1), make([]C.uint32_t, len(e.asks)+1)
	var done C.uint32_t
	if e.ck(C.yk_preemption_plan(e.h, C.uint32_t(n), &asks[0], &status[0], &node[0], &off[0], &victims[0],
		C.uint32_t(len(victims)), &done), "yk_preemption_plan") != nil {
		return nil
	}
	resp := &si.AllocationResponse{}
	for j := 0; j < int(done); j++ {
		if status[j] != C.YK_PP_PLANNED {
			continue
		}
		vs := victims[off[j]:off[j+1]]
		if C.yk_release(e.h, C.uint32_t(len(vs)), &vs[0]) != C.YK_OK {
			continue
		}
		for _, v := range vs {
			a := &e.asks[v]
			resp.Released = append(resp.Released, &si.AllocationRelease{ApplicationID: a.app, AllocationKey: a.key,
				TerminationType: si.TerminationType_PREEMPTED_BY_SCHEDULER, Message: "preempted by scheduler"})
			a.present = false
			delete(e.askIdx, a.key)
			e.freeAsks = append(e.freeAsks, uint32(v))
		}
		p := &e.asks[asks[j]]
		p.pinNode = uint32(node[j])
		_ = e.pushAsk(uint32(asks[j]), p, nil)
	}
	if len(resp.Released) == 0 {
		return nil
	}
	return resp
}

// preemptDaemons: the core's required-node preemption (yk_preemption_required_node, DESIGN.md §2 item 10), once per loop, for
// every DaemonSet ask that ended the cycle NOFIT / SKIPPED and has no plan, oldest blocked first.  There is no
// preemption.delay: the core's required-node path does not wait.  Only asks with dsNode go there -- never a guarantee-planned
// preemptor pinned through its required node.  The victims are released here and handed to the shim as preempted; the next
// cycle places the preemptor on its node.  Called with e.mu held; nil when nothing was preempted.
func (e *Engine) preemptDaemons() *si.AllocationResponse {
	var asks []C.uint32_t
	for i := range e.asks {
		a := &e.asks[i]
		if a.present && !a.foreign && !a.slow && a.dsNode != "" && !a.dsPlanned && !a.blocked.IsZero() {
			asks = append(asks, C.uint32_t(i))
		}
	}
	if len(asks) == 0 {
		return nil
	}
	sort.SliceStable(asks, func(x, y int) bool { return e.asks[asks[x]].blocked.Before(e.asks[asks[y]].blocked) })
	n := len(asks)
	status, off := make([]C.uint32_t, n), make([]C.uint32_t, n+1)
	victims := make([]C.uint32_t, len(e.asks)+1)
	var done C.uint32_t
	if e.ck(C.yk_preemption_required_node(e.h, C.uint32_t(n), &asks[0], &status[0], &off[0], &victims[0],
		C.uint32_t(len(victims)), &done), "yk_preemption_required_node") != nil {
		return nil
	}
	resp := &si.AllocationResponse{}
	for j := 0; j < int(done); j++ {
		if status[j] != C.YK_PP_PLANNED {
			continue
		}
		p := &e.asks[asks[j]]
		p.dsPlanned = true
		vs := victims[off[j]:off[j+1]]
		if C.yk_release(e.h, C.uint32_t(len(vs)), &vs[0]) != C.YK_OK {
			continue
		}
		for _, v := range vs {
			a := &e.asks[v]
			resp.Released = append(resp.Released, &si.AllocationRelease{ApplicationID: a.app, AllocationKey: a.key,
				TerminationType: si.TerminationType_PREEMPTED_BY_SCHEDULER,
				Message:         "preempting allocations to free up resources to run daemon set ask: " + p.key})
			a.present = false
			delete(e.askIdx, a.key)
			e.freeAsks = append(e.freeAsks, uint32(v))
		}
	}
	if len(resp.Released) == 0 {
		return nil
	}
	return resp
}

// collectStates: asks that ended the cycle NOFIT / SKIPPED and were not reported in that state yet ->
// UpdateContainerSchedulingState FAILED / SKIPPED (scheduler_callback.go:218-222 -> context.go:1232-1272: the FAILED
// state is what makes the shim mark the pod unschedulable and trigger the autoscaler)
func (e *Engine) collectStates() []*si.UpdateContainerSchedulingStateRequest {
	var idx []C.uint32_t
	for i := range e.asks {
		if a := &e.asks[i]; a.present && !a.foreign && a.lastState != C.YK_ST_ALLOCATED {
			idx = append(idx, C.uint32_t(i))
		}
	}
	if len(idx) == 0 {
		return nil
	}
	st := make([]C.uint8_t, len(idx))
	if C.yk_ask_states(e.h, C.uint32_t(len(idx)), &idx[0], &st[0]) != C.YK_OK {
		return nil
	}
	// the asks newly NOFIT get a per-cause reason, from one yk_filter_nodes call over all of them
	var nofit []C.uint32_t
	for j, i := range idx {
		if s := uint8(st[j]); s == C.YK_ST_NOFIT && s != e.asks[i].lastState {
			nofit = append(nofit, i)
		}
	}
	reason := map[C.uint32_t]string{}
	if len(nofit) > 0 {
		counts := make([]C.uint32_t, len(nofit)*C.YK_FILTER_SLOTS)
		if C.yk_filter_nodes(e.h, C.uint32_t(len(nofit)), &nofit[0], 1, 0, 0, nil, nil, &counts[0]) == C.YK_OK {
			for j, i := range nofit {
				reason[i] = failedReason(counts[j*C.YK_FILTER_SLOTS : (j+1)*C.YK_FILTER_SLOTS])
			}
		}
	}
	var out []*si.UpdateContainerSchedulingStateRequest
	for j, i := range idx {
		a := &e.asks[i]
		s := uint8(st[j])
		if s == a.lastState {
			continue
		}
		if s == C.YK_ST_NOFIT || s == C.YK_ST_SKIPPED {
			if a.lastState != C.YK_ST_NOFIT && a.lastState != C.YK_ST_SKIPPED {
				a.blocked = time.Now()
			}
		} else {
			a.blocked = time.Time{}
		}
		a.lastState = s
		switch s {
		case C.YK_ST_NOFIT:
			r, ok := reason[i]
			if !ok {
				r = "no node passes the predicates with enough resources"
			}
			out = append(out, &si.UpdateContainerSchedulingStateRequest{ApplicationID: a.app, AllocationKey: a.key,
				State: si.UpdateContainerSchedulingStateRequest_FAILED, Reason: r})
		case C.YK_ST_SKIPPED:
			out = append(out, &si.UpdateContainerSchedulingStateRequest{ApplicationID: a.app, AllocationKey: a.key,
				State: si.UpdateContainerSchedulingStateRequest_SKIPPED, Reason: "request exceeds the queue headroom"})
		}
	}
	return out
}

// failedReason: the FAILED reason of an unplaceable pod in the Kubernetes scheduler's style, from the yk_filter_nodes
// counts of its ask (one count per first failing step, summing to the node count), e.g.
// "0/5000 nodes are available: 3 node(s) were unschedulable, 4990 Insufficient resources, 7 node(s) had untolerated taint."
// Steps with no node are left out; a node too small (total), too full (available) or failing NodeResourcesFit counts as
// "Insufficient resources".
func failedReason(c []C.uint32_t) string {
	total := uint64(0)
	for _, x := range c {
		total += uint64(x)
	}
	parts := make([]string, 0, 8)
	add := func(n uint64, text string) {
		if n > 0 {
			parts = append(parts, fmt.Sprintf("%d %s", n, text))
		}
	}
	add(uint64(c[C.YK_FAIL_NODE_NOT_SCHEDULABLE]), "node(s) were unschedulable")
	add(uint64(c[C.YK_FAIL_TOTAL])+uint64(c[C.YK_FAIL_AVAILABLE])+uint64(c[C.YK_FAIL_RESOURCES]), "Insufficient resources")
	add(uint64(c[C.YK_FAIL_REQUEST_NOT_POSITIVE]), "request not positive")
	add(uint64(c[C.YK_FAIL_NODENAME]), "node(s) didn't match the requested node name")
	add(uint64(c[C.YK_FAIL_TAINT]), "node(s) had untolerated taint")
	add(uint64(c[C.YK_FAIL_AFFINITY]), "node(s) didn't match Pod's node affinity/selector")
	add(uint64(c[C.YK_FAIL_ABSENT]), "node(s) not found")
	add(uint64(c[C.YK_FILTER_RESERVED]), "node(s) were reserved")
	return fmt.Sprintf("0/%d nodes are available: %s.", total, strings.Join(parts, ", "))
}

// filterPage: one page of the engine's candidates for ask idx -- the nodes that pass every step the engine checks, in its
// node order, pass ranks skip .. skip+filterPageSize-1 -- as node names, and how many nodes pass in all.  Caller holds e.mu.
const filterPageSize = 64

func (e *Engine) filterPage(idx uint32, skip uint32) ([]string, uint32, bool) {
	page := make([]C.uint32_t, filterPageSize)
	var npass C.uint32_t
	i := C.uint32_t(idx)
	if C.yk_filter_nodes(e.h, 1, &i, 1, C.uint32_t(skip), filterPageSize, &page[0], &npass, nil) != C.YK_OK {
		return nil, 0, false
	}
	return e.pageNames(page), uint32(npass), true
}

func (e *Engine) pageNames(page []C.uint32_t) []string {
	names := make([]string, 0, len(page))
	for _, x := range page {
		if x == C.YK_NONE {
			break
		}
		names = append(names, e.nodes[x].name)
	}
	return names
}

// PreemptionNodes: the search half of a preemptor (PreemptionPredicates, predicate_manager.go:137-175, for every node at
// once).  victimKeys are the allocations the caller's preemption policy lets go for askKey, in its victim order; the engine
// knows where each is bound.  Returns the nodes where removing a prefix of those victims (in that order, per node) lets the
// ask fit, fit ranks skip .. skip+k-1 in the engine's node order, with the number of victims each needs, then how many
// nodes fit in all and the one needing the fewest (empty name when none fits).  Which allocations may be victims, and
// releasing them, stay with the caller.
func (e *Engine) PreemptionNodes(askKey string, victimKeys []string, skip, k uint32) (nodes []string, need []uint32, nFit uint32, best string, bestNeed uint32, err error) {
	e.mu.Lock()
	defer e.mu.Unlock()
	a, ok := e.askIdx[askKey]
	if !ok {
		return nil, nil, 0, "", 0, fmt.Errorf("ykgpu: unknown ask %s", askKey)
	}
	vic := make([]C.uint32_t, len(victimKeys)+1) // one spare element so &vic[0] is valid for an empty list
	for i, key := range victimKeys {
		v, ok := e.askIdx[key]
		if !ok {
			return nil, nil, 0, "", 0, fmt.Errorf("ykgpu: unknown victim %s", key)
		}
		vic[i] = C.uint32_t(v)
	}
	off := [2]C.uint32_t{0, C.uint32_t(len(victimKeys))}
	page := make([]C.uint32_t, k+1)
	cnt := make([]C.uint32_t, k+1)
	var fit, bn, bc C.uint32_t
	i := C.uint32_t(a)
	if err := e.ck(C.yk_preemption_nodes(e.h, 1, &i, &off[0], &vic[0], C.uint32_t(skip), C.uint32_t(k), &page[0], &cnt[0], &fit,
		&bn, &bc), "yk_preemption_nodes"); err != nil {
		return nil, nil, 0, "", 0, err
	}
	nodes = e.pageNames(page[:k])
	need = make([]uint32, len(nodes))
	for j := range need {
		need[j] = uint32(cnt[j])
	}
	if bn != C.YK_NONE {
		best = e.nodes[bn].name
	}
	return nodes, need, uint32(fit), best, uint32(bc), nil
}

// slowPath: pods whose predicates do not reduce to the bit sets.  Candidates are tried in the engine's node order
// (ascending float64 score, then NodeID) through the UNCHANGED Go path -- callback.Predicates ->
// Context.IsPodFitNode -> PredicateManager (scheduler_callback.go:196-198) -- and the first node that passes is pinned:
// the ask goes back to the engine naming that node (spec.nodeName semantics), everything else tolerated, so the next
// cycle re-checks the resources, commits and reports the binding like any other.
// An ask whose masks the dictionary encoded exactly (slow only for what needsGoPredicates names) walks only the nodes that
// pass the engine's own steps, a page of yk_filter_nodes at a time: every engine step is also a step of the
// PredicateManager (or of the core before it), so a node skipped there could never pass, and in the same order the first
// Go-passing candidate is the node the full walk reaches.  Every other slow-path ask walks every live node.
func (e *Engine) slowPath(cb api.ResourceManagerCallback, askIdxs []uint32) {
	if len(askIdxs) == 0 {
		return
	}
	e.mu.Lock()
	type job struct {
		idx   uint32
		key   string
		exact bool
		page  []string // first page of candidates (exact asks)
		npass uint32
	}
	jobs := make([]job, 0, len(askIdxs))
	var exactIdx []C.uint32_t
	for _, a := range askIdxs {
		if int(a) < len(e.asks) && e.asks[a].present {
			jobs = append(jobs, job{idx: a, key: e.asks[a].key, exact: e.asks[a].exact})
			if e.asks[a].exact {
				exactIdx = append(exactIdx, C.uint32_t(a))
			}
		}
	}
	// the first page of every exact ask in one call; if it fails they walk every node like the others
	if len(exactIdx) > 0 {
		first := make([]C.uint32_t, len(exactIdx)*filterPageSize)
		npass := make([]C.uint32_t, len(exactIdx))
		ok := C.yk_filter_nodes(e.h, C.uint32_t(len(exactIdx)), &exactIdx[0], 1, 0, filterPageSize, &first[0], &npass[0], nil) == C.YK_OK
		x := 0
		for j := range jobs {
			if !jobs[j].exact {
				continue
			}
			if ok {
				jobs[j].page = e.pageNames(first[x*filterPageSize : (x+1)*filterPageSize])
				jobs[j].npass = uint32(npass[x])
			} else {
				jobs[j].exact = false
			}
			x++
		}
	}
	walkAll := false
	for _, j := range jobs {
		walkAll = walkAll || !j.exact
	}
	var names []string // every live node in the engine's order, for the asks that walk them all
	if walkAll {
		live := make([]uint32, 0, len(e.nodes))
		for i := range e.nodes {
			if e.nodes[i].present && e.nodes[i].schedulable {
				live = append(live, uint32(i))
			}
		}
		ci := make([]C.uint32_t, len(live))
		for i, x := range live {
			ci[i] = C.uint32_t(x)
		}
		scores := make([]C.double, len(live))
		if len(live) > 0 {
			C.yk_node_scores(e.h, C.uint32_t(len(live)), &ci[0], &scores[0])
		}
		sort.Slice(live, func(a, b int) bool {
			if scores[a] != scores[b] {
				return scores[a] < scores[b]
			}
			return e.nodes[live[a]].name < e.nodes[live[b]].name
		})
		names = make([]string, len(live))
		for i, x := range live {
			names[i] = e.nodes[x].name
		}
	}
	e.mu.Unlock()
	for _, j := range jobs {
		chosen := ""
		if j.exact {
			chosen = e.walkCandidates(cb, j.idx, j.key, j.page, j.npass)
		} else {
			for _, node := range names {
				if cb.Predicates(&si.PredicatesArgs{AllocationKey: j.key, NodeID: node, Allocate: true}) == nil {
					chosen = node
					break
				}
			}
		}
		e.pinSlowAsk(j.idx, j.key, chosen)
	}
}

// walkCandidates: the first of the engine's candidates for an exact slow-path ask that the Go predicates accept, page by
// page (the first page is given), until one passes or the candidates run out; "" when none does
func (e *Engine) walkCandidates(cb api.ResourceManagerCallback, idx uint32, key string, page []string, npass uint32) string {
	for skip := uint32(0); ; {
		for _, node := range page {
			if cb.Predicates(&si.PredicatesArgs{AllocationKey: key, NodeID: node, Allocate: true}) == nil {
				return node
			}
		}
		skip += filterPageSize
		if skip >= npass {
			return ""
		}
		e.mu.Lock()
		var ok bool
		page, npass, ok = e.filterPage(idx, skip)
		e.mu.Unlock()
		if !ok {
			return ""
		}
	}
}

// pinSlowAsk: the chosen node goes back to the engine as the ask's node name; "" leaves the ask as it is
func (e *Engine) pinSlowAsk(idx uint32, key, chosen string) {
	e.mu.Lock()
	a := &e.asks[idx]
	if chosen == "" || !a.present || a.key != key {
		e.mu.Unlock()
		return // no node passes today: the ask stays SLOWPATH and is tried again next cycle
	}
	i, rn, all, zero, fl := C.uint32_t(idx), C.uint32_t(e.nodeIdx[chosen]), ^C.uint64_t(0), C.uint64_t(0), C.uint32_t(0)
	var rq [4]C.int64_t
	for k := 0; k < 4; k++ {
		rq[k] = C.int64_t(a.req[k])
	}
	app := C.uint32_t(e.appIdx[a.app])
	prio, seq := C.int32_t(0), C.int64_t(0) // first in its application: it was reached in order already
	C.yk_asks_upsert(e.h, 1, &i, &rq[0], &all, &zero, &zero, &prio, &seq, &app, &rn, &fl, nil)
	e.mu.Unlock()
	e.wake()
}
