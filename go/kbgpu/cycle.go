package kbgpu

/*
#include <stdlib.h>
#include "kbgpu.h"
*/
import "C"

import (
	"fmt"
	"sort"
	"unsafe"

	"github.com/golang/glog"
	v1 "k8s.io/api/core/v1"
	"k8s.io/apimachinery/pkg/types"
	"k8s.io/kubernetes/pkg/apis/scheduling"

	"github.com/kubernetes-sigs/kube-batch/pkg/scheduler/api"
	"github.com/kubernetes-sigs/kube-batch/pkg/scheduler/framework"
)

// Cycle runs the scheduler's configured action list ("reclaim, allocate, backfill, preempt", config/kube-batch-conf.yaml:1)
// as ONE kb_cycle on the device and hands every action shell its own slice of the result.
//
// Why one call: the actions share a *framework.Session* (scheduler.go:88-101) whose plugin state — drf shares, proportion's
// deserved / allocated, gang readiness — lives in closures the shim cannot read back.  A flatten-per-action design would have
// to re-derive that state from task statuses, which is not possible for proportion's `deserved` (computed once at
// OnSessionOpen).  So the FIRST kbgpu action that runs in a session flattens it as opened, runs the whole list on the GPU,
// and every action's Execute only REPLAYS its decisions through the unchanged ssn.Evict / ssn.Pipeline / ssn.Allocate /
// framework.Statement, keeping the Go session, the event handlers and the cache in step.
//
// UNVERIFIED BY A COMPILER HERE (no Go toolchain in the build image): reviewed source.
type Cycle struct {
	engine  *Engine
	actions []string // the configured order, e.g. {"reclaim", "allocate", "backfill", "preempt"}

	uid      types.UID // session the cached result belongs to
	flat     *Flat
	running  []*api.TaskInfo
	dec      []Decision
	evicted  []bool
	order    []uint32
	bounds   [][2]uint32
	failed   error
}

var actionID = map[string]C.uint8_t{"reclaim": C.KB_ACT_RECLAIM, "allocate": C.KB_ACT_ALLOCATE, "backfill": C.KB_ACT_BACKFILL, "preempt": C.KB_ACT_PREEMPT}

// NewCycle: `actions` must be the scheduler configuration's action list restricted to the four built-ins, in order.
func NewCycle(e *Engine, actions []string) (*Cycle, error) {
	for i, a := range actions {
		if _, ok := actionID[a]; !ok {
			return nil, fmt.Errorf("kbgpu: unknown action %q", a)
		}
		for _, prev := range actions[:i] {
			if prev == a { // replay finds an action's slice of the result by its name
				return nil, fmt.Errorf("kbgpu: action %q is listed twice", a)
			}
		}
	}
	return &Cycle{engine: e, actions: actions}, nil
}

// flattenRunning lists the Running tasks one by one (kb_running): what reclaim / preempt walk as `n.Tasks`.
type runningFlat struct {
	node, job, present, uidRank, flags []uint32
	resreq                             []float64 // [R][n]
	prio                               []int32
	ctime                              []int64
	waiting                            []int32 // [J]
	affGroupOff, affGroup              []uint32 // [n+1] + the counter groups of each Running task
}

func (c *Cycle) flattenRunning(ssn *framework.Session, f *Flat) *runningFlat {
	jidx := make(map[api.JobID]uint32, len(f.JobIDs))
	for i, id := range f.JobIDs {
		jidx[id] = uint32(i)
	}
	c.running = c.running[:0]
	var nodeOf []uint32
	for ni, name := range f.NodeNames {
		for _, t := range ssn.Nodes[name].Tasks {
			if t.Status != api.Running { // reclaim.go:127, preempt.go:105
				continue
			}
			if _, ok := jidx[t.Job]; !ok { // reclaim.go:131: tasks of unknown jobs are never candidates
				continue
			}
			// reclaim.go:135-136: a clone, so that the node's own copy still holds Running when ssn.Evict / Statement.Evict
			// take it off the node (node_info.go:217-245); evicting the node's copy itself would leave Releasing unchanged
			c.running = append(c.running, t.Clone())
			nodeOf = append(nodeOf, uint32(ni))
		}
	}
	n := len(c.running)
	uids := make([]string, n)
	for i, t := range c.running {
		uids[i] = string(t.UID)
	}
	sort.Strings(uids)
	rank := make(map[string]uint32, n)
	for i, u := range uids {
		rank[u] = uint32(i)
	}
	R := int(f.R)
	r := &runningFlat{node: make([]uint32, max1(n)), job: make([]uint32, max1(n)), present: make([]uint32, max1(n)),
		uidRank: make([]uint32, max1(n)), flags: make([]uint32, max1(n)), resreq: make([]float64, R*max1(n)),
		prio: make([]int32, max1(n)), ctime: make([]int64, max1(n)), waiting: make([]int32, max1(len(f.JobIDs))),
		affGroupOff: make([]uint32, n+1)}
	for i, t := range c.running {
		r.node[i] = nodeOf[i]
		r.job[i] = jidx[t.Job]
		r.present[i] = f.resourceVec(t.Resreq, r.resreq, n, i)
		r.prio[i] = t.Priority
		r.uidRank[i] = rank[string(t.UID)]
		if t.Pod != nil {
			r.ctime[i] = t.Pod.CreationTimestamp.UnixNano()
			cn := t.Pod.Spec.PriorityClassName // conformance.go:45-53
			if cn == scheduling.SystemClusterCritical || cn == scheduling.SystemNodeCritical || t.Namespace == v1.NamespaceSystem {
				r.flags[i] |= uint32(C.KB_RUNNING_CRITICAL)
			}
			if f.podAff != nil && f.podAff.members[t.Pod] { // its eviction takes it out of util.PodLister: kbgpu.h KB_RUNNING_AFF_MEMBER
				r.flags[i] |= uint32(C.KB_RUNNING_AFF_MEMBER)
			}
		}
		// its counter groups (kb_running.aff_group_off / aff_group, builder.py meta["running_aff_groups"]): always filled, so the engine
		// keeps the member bits exact when it is evicted instead of withholding the cycle
		if f.podAff != nil && t.Pod != nil {
			r.affGroup = append(r.affGroup, f.podAff.memberGroups[t.Pod]...)
		}
		r.affGroupOff[i+1] = uint32(len(r.affGroup))
	}
	for j, id := range f.JobIDs { // WaitingTaskNum (job_info.go:396-405): 0 unless an earlier action pipelined tasks
		r.waiting[j] = int32(len(ssn.Jobs[id].TaskStatusIndex[api.Pipelined]))
	}
	return r
}

// ensure runs the whole list once per session.
func (c *Cycle) ensure(ssn *framework.Session) error {
	if c.uid == ssn.UID {
		return c.failed
	}
	if c.flat != nil {
		c.flat.Free()
		c.flat = nil
	}
	c.uid = ssn.UID
	c.failed = c.run(ssn)
	return c.failed
}

func (c *Cycle) run(ssn *framework.Session) error {
	flat, err := Flatten(ssn)
	if err != nil {
		return err
	}
	c.flat = flat
	if err := c.engine.Load(flat); err != nil {
		return err
	}
	rf := c.flattenRunning(ssn, flat)
	var a arena
	defer a.free()
	snap := (*C.kb_snapshot)(C.calloc(1, C.size_t(unsafe.Sizeof(C.kb_snapshot{}))))
	defer C.free(unsafe.Pointer(snap))
	flat.cSnapshot(snap, &a)
	run := (*C.kb_running)(C.calloc(1, C.size_t(unsafe.Sizeof(C.kb_running{}))))
	defer C.free(unsafe.Pointer(run))
	run.n = C.uint32_t(len(c.running))
	run.node, run.job, run.res_present = a.u32(rf.node), a.u32(rf.job), a.u32(rf.present)
	run.resreq, run.prio, run.ctime = a.f64(rf.resreq), a.i32(rf.prio), a.i64(rf.ctime)
	run.uid_rank, run.flags, run.job_waiting0 = a.u32(rf.uidRank), a.u32(rf.flags), a.i32(rf.waiting)
	run.aff_group_off, run.aff_group = a.u32(rf.affGroupOff), a.u32(append(rf.affGroup, 0)) // a.u32 needs one element
	evicts := false // only reclaim and preempt read the Running tasks: without them a session the victim walk cannot run is not refused
	for _, name := range c.actions {
		evicts = evicts || name == "reclaim" || name == "preempt"
	}
	if evicts {
		if rc := C.kb_session_load_running(c.engine.h, snap, run); rc != 0 {
			if rc == C.KB_E_UNSUPPORTED_FEATURE {
				return &ErrUnsupported{C.GoString(C.kb_last_error(c.engine.h))}
			}
			return c.engine.err("kb_session_load_running", rc)
		}
	}
	acts := make([]C.uint8_t, len(c.actions))
	for i, name := range c.actions {
		acts[i] = actionID[name]
	}
	T, n := len(flat.Tasks), len(c.running)
	raw := make([]C.kb_decision, T+1)
	ev := make([]C.uint8_t, n+1)
	ord := make([]C.uint32_t, n+1)
	bnd := make([]C.uint32_t, 2*len(acts)+2)
	var st C.kb_stats
	if rc := C.kb_cycle(c.engine.h, &acts[0], C.uint32_t(len(acts)), (*C.kb_decision)(unsafe.Pointer(&raw[0])), &ev[0], &ord[0], &bnd[0], &st); rc != 0 {
		if rc == C.KB_E_UNSUPPORTED_FEATURE {
			return &ErrUnsupported{C.GoString(C.kb_last_error(c.engine.h))}
		}
		return c.engine.err("kb_cycle", rc)
	}
	c.dec = make([]Decision, T)
	for i := range c.dec {
		c.dec[i] = Decision{Node: int32(raw[i].node), Kind: uint8(raw[i].kind), Dispatched: raw[i].dispatched != 0,
			Step: uint32(raw[i].step), DispatchStep: uint32(raw[i].dispatch_step)}
	}
	c.evicted, c.order = make([]bool, n), make([]uint32, n)
	for i := 0; i < n; i++ {
		c.evicted[i], c.order[i] = ev[i] != 0, uint32(ord[i])
	}
	c.bounds = make([][2]uint32, len(acts))
	for i := range acts {
		c.bounds[i] = [2]uint32{uint32(bnd[2*i]), uint32(bnd[2*i+1])}
	}
	return nil
}

// replay applies the decisions action `name` made, in the order the reference would have made the calls.
func (c *Cycle) replay(ssn *framework.Session, name string) {
	idx := -1
	for i, a := range c.actions {
		if a == name {
			idx = i
		}
	}
	if idx < 0 {
		glog.Errorf("kbgpu: action %q is not part of the configured cycle %v", name, c.actions)
		return
	}
	var lo [2]uint32
	if idx > 0 {
		lo = c.bounds[idx-1]
	}
	hi := c.bounds[idx]
	// evictions of this action, in cache.Evict order
	var evs []int
	for i, e := range c.evicted {
		if e && c.order[i] >= lo[1] && c.order[i] < hi[1] {
			evs = append(evs, i)
		}
	}
	sort.Slice(evs, func(a, b int) bool { return c.order[evs[a]] < c.order[evs[b]] })
	// placements of this action, in step order
	var pls []int
	for i, d := range c.dec {
		if (d.Kind == 1 || d.Kind == 2) && d.Step != 0xFFFFFFFF && d.Step >= lo[0] && d.Step < hi[0] {
			pls = append(pls, i)
		}
	}
	sort.Slice(pls, func(a, b int) bool { return c.dec[pls[a]].Step < c.dec[pls[b]].Step })
	switch name {
	case "preempt":
		// the engine only reports committed statements (preempt.go:121-131); one Statement replays them: evictions first, so that
		// node.Releasing covers the pipelined tasks (node_info.go:190-192), then Commit sends the evictions to the cache
		stmt := ssn.Statement()
		for _, i := range evs {
			if err := stmt.Evict(c.running[i], "preempt"); err != nil {
				glog.Errorf("kbgpu: replay of the eviction of %v failed: %v", c.running[i].UID, err)
			}
		}
		for _, i := range pls {
			if err := stmt.Pipeline(c.flat.Tasks[i], c.flat.NodeNames[c.dec[i].Node]); err != nil {
				glog.Errorf("kbgpu: replay of the pipeline of %v failed: %v", c.flat.Tasks[i].UID, err)
			}
		}
		stmt.Commit()
	case "reclaim":
		// reclaim.go:157-185 interleaves: the victims of one reclaimer, then its Pipeline.  Replaying all evictions of the action
		// first and the pipelines after them leaves the same session state (evictions only add to Releasing).
		for _, i := range evs {
			if err := ssn.Evict(c.running[i], "reclaim"); err != nil {
				glog.Errorf("kbgpu: replay of the eviction of %v failed: %v", c.running[i].UID, err)
			}
		}
		for _, i := range pls {
			if err := ssn.Pipeline(c.flat.Tasks[i], c.flat.NodeNames[c.dec[i].Node]); err != nil {
				glog.Errorf("kbgpu: replay of the pipeline of %v failed: %v", c.flat.Tasks[i].UID, err)
			}
		}
	default: // allocate, backfill
		for _, i := range pls {
			task, node := c.flat.Tasks[i], c.flat.NodeNames[c.dec[i].Node]
			var err error
			if c.dec[i].Kind == 1 {
				err = ssn.Allocate(task, node) // dispatches on its own when ssn.JobReady (session.go:277-285)
			} else {
				err = ssn.Pipeline(task, node)
			}
			if err != nil {
				glog.Errorf("kbgpu: replay of task %v on %v failed: %v", task.UID, node, err)
			}
		}
		// backfill's phantom tasks (Allocated on no node, step none: session.go:241-262) are not replayed: the reference itself
		// calls that state "will be corrected in next scheduling loop"
	}
}

// action is the drop-in shell of one of the four actions: same Name(), same framework.Action interface
// (framework/interface.go:20-32); Fallback is the ORIGINAL action, run for the cycles libkbgpu refuses.
type action struct {
	name     string
	cycle    *Cycle
	Fallback framework.Action
}

func (a *action) Name() string    { return a.name }
func (a *action) Initialize()     {}
func (a *action) UnInitialize()   {}
func (a *action) Execute(ssn *framework.Session) {
	if err := a.cycle.ensure(ssn); err != nil {
		fallBack(a.Fallback, ssn, err)
		return
	}
	a.cycle.replay(ssn, a.name)
}

// Actions returns the four shells for framework.RegisterAction (actions/factory.go:28-33).  fallbacks: the original actions by name.
func (c *Cycle) Actions(fallbacks map[string]framework.Action) []framework.Action {
	var out []framework.Action
	for _, name := range []string{"reclaim", "allocate", "backfill", "preempt"} {
		out = append(out, &action{name: name, cycle: c, Fallback: fallbacks[name]})
	}
	return out
}
