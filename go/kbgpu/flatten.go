package kbgpu

/*
#include <stdlib.h>
#include <string.h>
#include "kbgpu.h"
*/
import "C"

import (
	"fmt"
	"sort"
	"unsafe"

	v1 "k8s.io/api/core/v1"
	"k8s.io/apimachinery/pkg/fields"
	"k8s.io/apimachinery/pkg/labels"
	v1helper "k8s.io/kubernetes/pkg/apis/core/v1/helper"
	v1qos "k8s.io/kubernetes/pkg/apis/core/v1/helper/qos"
	priorityutil "k8s.io/kubernetes/pkg/scheduler/algorithm/priorities/util"

	"github.com/kubernetes-sigs/kube-batch/pkg/scheduler/api"
	"github.com/kubernetes-sigs/kube-batch/pkg/scheduler/conf"
	"github.com/kubernetes-sigs/kube-batch/pkg/scheduler/framework"
)

// Flat is the SoA form of ssn.Jobs / ssn.Nodes / ssn.Queues that kb_snapshot points into (include/kbgpu.h).
// The executable specification of every field is kube_batch_b200/builder.py::SessionBuilder.flatten and its C++ twin
// kube_batch_b200/host/kbhost.hpp::Flatten (cross-checked field by field in tests/test_host_cpp.py); this file is the
// same computation over the real Go objects.  UNVERIFIED BY A COMPILER HERE: the build image has no Go toolchain
// (INTEGRATION.md), so treat it as reviewed source, not as tested code.
type Flat struct {
	R, W, N, T, J, Q uint32
	Dims             []v1.ResourceName // dim 0 cpu, 1 memory, 2.. scalar names (sorted)
	NodeNames        []string          // canonical node order (ascending Name)
	Tasks            []*api.TaskInfo   // snapshot task index -> task
	JobIDs           []api.JobID
	QueueIDs         []api.QueueID

	nodeIdle, nodeReleasing, nodeUsed, nodeAllocatable []float64 // [R][N]
	nodeAllocPresent, nodeFlags                        []uint32
	nodeAllocCPU, nodeAllocMem, nodeNzCPU, nodeNzMem   []int64
	nodePods, nodeMaxPods                              []int32
	nodeLabels, nodeTaints, nodePorts                  []uint64 // [W][N]

	taskInitreq, taskResreq                                     []float64 // [R][T]
	taskResPresent, taskNAff, taskFlags, taskUIDRank, taskNPref []uint32
	taskNzCPU, taskNzMem, taskCtime                             []int64
	taskSelReq, taskTol, taskPortOwn, taskPortConflict          []uint64 // [W][T]
	taskAff                                                     []uint64 // [KB_MAX_AFF_TERMS][W][T]
	taskPref                                                    []uint64 // [KB_MAX_PREF_TERMS][W][T]
	taskPrefWeight                                              []int32  // [KB_MAX_PREF_TERMS][T]
	taskPrio                                                    []int32

	jobTaskOff, jobAlloc0Present, jobQueue []uint32
	jobMinAvail, jobReady0, jobPrio        []int32
	jobAlloc0                              []float64 // [R][J]
	jobCtime, queueCtime                   []int64
	queueWeight                            []int32

	snapFlags uint32  // KB_SNAPSHOT_*
	podAff    *podAff // inter-pod (anti)affinity tables (podaffinity.go), nil when no pod of the session carries terms

	// C-side copy of the tier configuration (strings, option and tier arrays), released by Free
	cstrings []*C.char
	cTiers   *C.kb_tier
	nTiers   int
}

const (
	maxR         = 32 // KB_MAX_R
	maxW         = 16 // KB_MAX_W
	narrowR      = 8  // KB_NARROW_R (kb_core.h): sessions with more dimensions take at most narrowW words
	narrowW      = 4  // KB_NARROW_W
	maxAffTerms  = 4  // KB_MAX_AFF_TERMS
	maxPrefTerms = 4  // KB_MAX_PREF_TERMS
)

var builtin = map[string]bool{"priority": true, "gang": true, "drf": true, "predicates": true, "proportion": true,
	"nodeorder": true, "conformance": true}

// ErrUnsupported marks sessions libkbgpu refuses by design (non built-in plugin, inter-pod affinity, too many atoms):
// the action then runs the original Go implementation for this cycle instead (allocate.go: fallback).
type ErrUnsupported struct{ Why string }

func (e *ErrUnsupported) Error() string { return "kbgpu: unsupported session: " + e.Why }

// reqAtom is one node-selector requirement evaluated ONCE per node: (key, operator, values) of a nodeSelector pair, a
// required / preferred node-affinity MatchExpression, or a MatchFields requirement on metadata.name.
type reqAtom struct {
	field    bool
	key      string
	operator v1.NodeSelectorOperator
	values   string // values joined with '\x00' (order kept: identical requirements written identically share the atom)
}

type atomTable struct {
	ids  map[reqAtom]uint32
	reqs []v1.NodeSelectorRequirement
	fld  []bool
}

func (a *atomTable) of(req v1.NodeSelectorRequirement, field bool) uint32 {
	k := reqAtom{field: field, key: req.Key, operator: req.Operator}
	for i, v := range req.Values {
		if i > 0 {
			k.values += "\x00"
		}
		k.values += v
	}
	if id, ok := a.ids[k]; ok {
		return id
	}
	id := uint32(len(a.reqs))
	a.ids[k] = id
	a.reqs = append(a.reqs, req)
	a.fld = append(a.fld, field)
	return id
}

// never is an atom no node satisfies: a required term without expressions matches nothing
// (v1helper.MatchNodeSelectorTerms skips it), so a pod whose every term is empty fits nowhere; a preferred term without
// expressions adds its weight nowhere.
func (a *atomTable) never() uint32 {
	return a.of(v1.NodeSelectorRequirement{Key: "\x00never", Operator: v1.NodeSelectorOpIn, Values: []string{"\x00"}}, false)
}

// holds evaluates atom i on a node exactly like the vendored predicate does
// (predicates.go:880-968: NodeSelectorRequirementsAsSelector / NodeSelectorRequirementsAsFieldSelector).
func (a *atomTable) holds(i int, node *v1.Node) bool {
	req := []v1.NodeSelectorRequirement{a.reqs[i]}
	if a.fld[i] {
		sel, err := v1helper.NodeSelectorRequirementsAsFieldSelector(req)
		if err != nil {
			return false
		}
		return sel.Matches(fields.Set{"metadata.name": node.Name})
	}
	sel, err := v1helper.NodeSelectorRequirementsAsSelector(req)
	if err != nil {
		return false
	}
	return sel.Matches(labels.Set(node.Labels))
}

type taintAtom struct{ key, value, effect string }
type portAtom struct {
	ip, proto string
	port      int32
}

func sanitizePort(ip string, proto v1.Protocol, port int32) portAtom { // nodeinfo/host_ports.go:52-61
	if ip == "" {
		ip = "0.0.0.0"
	}
	if proto == "" {
		proto = v1.ProtocolTCP
	}
	return portAtom{ip, string(proto), port}
}

func portsConflict(a, b portAtom) bool { // HostPortInfo.CheckConflict, host_ports.go:96-125
	if a.proto != b.proto || a.port != b.port {
		return false
	}
	return a.ip == b.ip || a.ip == "0.0.0.0" || b.ip == "0.0.0.0"
}

func hostPorts(pod *v1.Pod) []portAtom {
	var out []portAtom
	for i := range pod.Spec.Containers {
		for _, p := range pod.Spec.Containers[i].Ports {
			if p.HostPort > 0 {
				out = append(out, sanitizePort(p.HostIP, p.Protocol, p.HostPort))
			}
		}
	}
	return out
}

// podNonzero is getNonZeroRequests (resource_allocation.go:127-141) == what nodeinfo.calculateResource adds per pod.
func podNonzero(pod *v1.Pod) (cpu, mem int64) {
	for i := range pod.Spec.Containers {
		c, m := priorityutil.GetNonzeroRequests(&pod.Spec.Containers[i].Resources.Requests)
		cpu += c
		mem += m
	}
	return
}

func setbit(a []uint64, stride, i int, atom uint32) {
	a[int(atom/64)*stride+i] |= uint64(1) << (atom % 64)
}

func (f *Flat) dim(name v1.ResourceName) int {
	for i, d := range f.Dims {
		if d == name {
			return i
		}
	}
	return -1
}

// resourceVec writes api.Resource r into column i of a [R][stride] array and returns the scalar-presence mask.
func (f *Flat) resourceVec(r *api.Resource, out []float64, stride, i int) uint32 {
	if r == nil {
		return 0
	}
	out[0*stride+i] = r.MilliCPU
	out[1*stride+i] = r.Memory
	var present uint32
	for name, v := range r.ScalarResources {
		k := f.dim(name)
		out[k*stride+i] = v
		present |= 1 << uint(k)
	}
	return present
}

func max1(n int) int {
	if n < 1 {
		return 1
	}
	return n
}

// Flatten walks the session once.  It returns *ErrUnsupported for sessions the GPU path cannot honour.
func Flatten(ssn *framework.Session) (*Flat, error) {
	for _, tier := range ssn.Tiers {
		for _, p := range tier.Plugins {
			if !builtin[p.Name] {
				return nil, &ErrUnsupported{fmt.Sprintf("plugin %q is not a built-in: its closures cannot run on the device", p.Name)}
			}
		}
	}
	f := &Flat{}
	// ---- canonical orders (SURVEY.md §8c rules 1 and 4) ----
	for name := range ssn.Nodes {
		f.NodeNames = append(f.NodeNames, name)
	}
	sort.Strings(f.NodeNames)
	queueIDs := make([]string, 0, len(ssn.Queues))
	for id := range ssn.Queues {
		queueIDs = append(queueIDs, string(id))
	}
	sort.Strings(queueIDs)
	qidx := make(map[api.QueueID]uint32, len(queueIDs))
	for i, id := range queueIDs {
		f.QueueIDs = append(f.QueueIDs, api.QueueID(id))
		qidx[api.QueueID(id)] = uint32(i)
	}
	jobIDs := make([]string, 0, len(ssn.Jobs))
	for id, job := range ssn.Jobs {
		if _, ok := qidx[job.Queue]; !ok { // allocate.go:56-60 skips jobs whose queue is unknown
			continue
		}
		jobIDs = append(jobIDs, string(id))
	}
	sort.Strings(jobIDs)
	for _, id := range jobIDs {
		f.JobIDs = append(f.JobIDs, api.JobID(id))
	}
	N, J, Q := len(f.NodeNames), len(f.JobIDs), len(f.QueueIDs)

	// ---- pending tasks grouped by job (allocate.go:112), UID ranks ----
	f.jobTaskOff = make([]uint32, J+1)
	var uids []string
	for j, id := range f.JobIDs {
		job := ssn.Jobs[id]
		pend := make([]*api.TaskInfo, 0, len(job.TaskStatusIndex[api.Pending]))
		for _, t := range job.TaskStatusIndex[api.Pending] {
			pend = append(pend, t)
		}
		sort.Slice(pend, func(a, b int) bool { return pend[a].UID < pend[b].UID })
		for _, t := range pend {
			f.Tasks = append(f.Tasks, t)
			uids = append(uids, string(t.UID))
		}
		f.jobTaskOff[j+1] = uint32(len(f.Tasks))
	}
	T := len(f.Tasks)
	sort.Strings(uids)
	uidRank := make(map[string]uint32, T)
	for i, u := range uids {
		uidRank[u] = uint32(i)
	}
	if len(uidRank) != T {
		return nil, fmt.Errorf("kbgpu: duplicate task UIDs in the session")
	}

	// ---- inter-pod (anti)affinity (predicate step 10 / InterPodAffinityPriority): flattened at the end of this function into
	//      kb_pod_affinity (podaffinity.go) once the task flags exist ----

	// ---- resource dims ----
	scalars := map[v1.ResourceName]bool{}
	for _, n := range ssn.Nodes {
		for name := range n.Allocatable.ScalarResources {
			scalars[name] = true
		}
	}
	for _, job := range ssn.Jobs {
		for _, t := range job.Tasks {
			for name := range t.Resreq.ScalarResources {
				scalars[name] = true
			}
			for name := range t.InitResreq.ScalarResources {
				scalars[name] = true
			}
		}
	}
	names := make([]string, 0, len(scalars))
	for name := range scalars {
		names = append(names, string(name))
	}
	sort.Strings(names)
	f.Dims = []v1.ResourceName{v1.ResourceCPU, v1.ResourceMemory}
	for _, s := range names {
		f.Dims = append(f.Dims, v1.ResourceName(s))
	}
	R := len(f.Dims)
	if R > maxR {
		return nil, &ErrUnsupported{fmt.Sprintf("%d resource dimensions > KB_MAX_R (%d)", R, maxR)}
	}

	// ---- atoms ----
	atoms := &atomTable{ids: map[reqAtom]uint32{}}
	type taskTerms struct {
		sel   []uint32
		aff   [][]uint32
		pref  [][]uint32
		prefW []int32
	}
	terms := make([]taskTerms, T)
	for ti, t := range f.Tasks {
		spec := &t.Pod.Spec
		keys := make([]string, 0, len(spec.NodeSelector))
		for k := range spec.NodeSelector {
			keys = append(keys, k)
		}
		sort.Strings(keys)
		for _, k := range keys { // predicates.go:927-935: labels.SelectorFromSet(pod.Spec.NodeSelector)
			terms[ti].sel = append(terms[ti].sel, atoms.of(v1.NodeSelectorRequirement{Key: k, Operator: v1.NodeSelectorOpIn, Values: []string{spec.NodeSelector[k]}}, false))
		}
		if spec.Affinity == nil || spec.Affinity.NodeAffinity == nil {
			continue
		}
		na := spec.Affinity.NodeAffinity
		if req := na.RequiredDuringSchedulingIgnoredDuringExecution; req != nil { // predicates.go:944-968
			for _, term := range req.NodeSelectorTerms {
				if len(term.MatchExpressions) == 0 && len(term.MatchFields) == 0 {
					continue // matches nothing
				}
				var as []uint32
				for _, e := range term.MatchExpressions {
					as = append(as, atoms.of(e, false))
				}
				for _, e := range term.MatchFields {
					as = append(as, atoms.of(e, true))
				}
				terms[ti].aff = append(terms[ti].aff, as)
			}
			if len(terms[ti].aff) == 0 {
				terms[ti].aff = [][]uint32{{atoms.never()}}
			}
			if len(terms[ti].aff) > maxAffTerms {
				return nil, &ErrUnsupported{fmt.Sprintf("pod %s/%s has %d required node-affinity terms > KB_MAX_AFF_TERMS", t.Namespace, t.Name, len(terms[ti].aff))}
			}
		}
		for _, p := range na.PreferredDuringSchedulingIgnoredDuringExecution { // node_affinity.go:34-77
			if p.Weight == 0 {
				continue
			}
			var as []uint32
			for _, e := range p.Preference.MatchExpressions { // MatchFields are ignored by the priority (node_affinity.go:52-56)
				as = append(as, atoms.of(e, false))
			}
			if len(as) == 0 { // NodeSelectorRequirementsAsSelector(nil) is labels.Nothing() (helpers.go:205-208): the term matches no node
				as = []uint32{atoms.never()}
			}
			terms[ti].pref = append(terms[ti].pref, as)
			terms[ti].prefW = append(terms[ti].prefW, p.Weight)
		}
		if len(terms[ti].pref) > maxPrefTerms {
			return nil, &ErrUnsupported{fmt.Sprintf("pod %s/%s has %d preferred node-affinity terms > KB_MAX_PREF_TERMS", t.Namespace, t.Name, len(terms[ti].pref))}
		}
	}
	taints := map[taintAtom]uint32{}
	var taintList []v1.Taint
	for _, name := range f.NodeNames {
		n := ssn.Nodes[name]
		if n.Node == nil {
			continue
		}
		for _, t := range n.Node.Spec.Taints { // predicates.go:1596-1624: only NoSchedule / NoExecute taints filter
			if t.Effect != v1.TaintEffectNoSchedule && t.Effect != v1.TaintEffectNoExecute {
				continue
			}
			k := taintAtom{t.Key, t.Value, string(t.Effect)}
			if _, ok := taints[k]; !ok {
				taints[k] = uint32(len(taintList))
				taintList = append(taintList, t)
			}
		}
	}
	ports := map[portAtom]uint32{}
	var portList []portAtom
	addPorts := func(pod *v1.Pod) {
		for _, p := range hostPorts(pod) {
			if _, ok := ports[p]; !ok {
				ports[p] = uint32(len(portList))
				portList = append(portList, p)
			}
		}
	}
	for _, t := range f.Tasks {
		addPorts(t.Pod)
	}
	for _, name := range f.NodeNames {
		for _, t := range ssn.Nodes[name].Tasks {
			if t.Pod != nil {
				addPorts(t.Pod)
			}
		}
	}
	need := len(atoms.reqs)
	if len(taintList) > need {
		need = len(taintList)
	}
	if len(portList) > need {
		need = len(portList)
	}
	W := (max1(need) + 63) / 64
	if W > maxW {
		return nil, &ErrUnsupported{fmt.Sprintf("%d label / taint / port atoms > 64 x KB_MAX_W (%d)", need, maxW)}
	}
	if R > narrowR && W > narrowW {
		return nil, &ErrUnsupported{fmt.Sprintf("%d resource dimensions > KB_NARROW_R (%d) with %d atoms > 64 x KB_NARROW_W (%d)", R, narrowR, need, narrowW)}
	}
	f.R, f.W, f.N, f.T, f.J, f.Q = uint32(R), uint32(W), uint32(N), uint32(T), uint32(J), uint32(Q)

	// ---- nodes ----
	f.nodeIdle = make([]float64, R*max1(N))
	f.nodeReleasing = make([]float64, R*max1(N))
	f.nodeUsed = make([]float64, R*max1(N))
	f.nodeAllocatable = make([]float64, R*max1(N))
	f.nodeAllocPresent = make([]uint32, max1(N))
	f.nodeFlags = make([]uint32, max1(N))
	f.nodeAllocCPU = make([]int64, max1(N))
	f.nodeAllocMem = make([]int64, max1(N))
	f.nodeNzCPU = make([]int64, max1(N))
	f.nodeNzMem = make([]int64, max1(N))
	f.nodePods = make([]int32, max1(N))
	f.nodeMaxPods = make([]int32, max1(N))
	f.nodeLabels = make([]uint64, W*max1(N))
	f.nodeTaints = make([]uint64, W*max1(N))
	f.nodePorts = make([]uint64, W*max1(N))
	for i, name := range f.NodeNames {
		n := ssn.Nodes[name]
		f.resourceVec(n.Idle, f.nodeIdle, N, i)
		f.resourceVec(n.Releasing, f.nodeReleasing, N, i)
		f.resourceVec(n.Used, f.nodeUsed, N, i)
		f.nodeAllocPresent[i] = f.resourceVec(n.Allocatable, f.nodeAllocatable, N, i)
		f.nodeMaxPods[i] = int32(n.Allocatable.MaxTaskNum)
		f.nodePods[i] = int32(len(n.Tasks)) // predicates.go:127
		for _, t := range n.Tasks {         // schedulernodeinfo.NewNodeInfo(node.Pods()...) (scheduler_helper.go:224)
			if t.Pod == nil {
				continue
			}
			c, m := podNonzero(t.Pod)
			f.nodeNzCPU[i] += c
			f.nodeNzMem[i] += m
			for _, p := range hostPorts(t.Pod) {
				setbit(f.nodePorts, N, i, ports[p])
			}
		}
		node := n.Node
		if node == nil {
			f.nodeFlags[i] = uint32(C.KB_NODE_NOT_READY)
			continue
		}
		// nodeinfo.SetNode: allocatableResource = NewResource(node.Status.Allocatable)
		f.nodeAllocCPU[i] = node.Status.Allocatable.Cpu().MilliValue()
		f.nodeAllocMem[i] = node.Status.Allocatable.Memory().Value()
		var fl uint32
		for _, c := range node.Status.Conditions { // predicates.go:1675-1698, 1633-1671
			switch c.Type {
			case v1.NodeReady:
				if c.Status != v1.ConditionTrue {
					fl |= uint32(C.KB_NODE_NOT_READY)
				}
			case v1.NodeNetworkUnavailable:
				if c.Status != v1.ConditionFalse {
					fl |= uint32(C.KB_NODE_NET_UNAVAILABLE)
				}
			case v1.NodeMemoryPressure:
				if c.Status == v1.ConditionTrue {
					fl |= uint32(C.KB_NODE_MEM_PRESSURE)
				}
			case v1.NodeDiskPressure:
				if c.Status == v1.ConditionTrue {
					fl |= uint32(C.KB_NODE_DISK_PRESSURE)
				}
			case v1.NodePIDPressure:
				if c.Status == v1.ConditionTrue {
					fl |= uint32(C.KB_NODE_PID_PRESSURE)
				}
			}
		}
		if node.Spec.Unschedulable {
			fl |= uint32(C.KB_NODE_UNSCHEDULABLE)
		}
		f.nodeFlags[i] = fl
		for a := range atoms.reqs {
			if atoms.holds(a, node) {
				setbit(f.nodeLabels, N, i, uint32(a))
			}
		}
		for _, t := range node.Spec.Taints {
			if a, ok := taints[taintAtom{t.Key, t.Value, string(t.Effect)}]; ok {
				setbit(f.nodeTaints, N, i, a)
			}
		}
	}

	// ---- pending tasks ----
	f.taskInitreq = make([]float64, R*max1(T))
	f.taskResreq = make([]float64, R*max1(T))
	f.taskResPresent = make([]uint32, max1(T))
	f.taskNAff = make([]uint32, max1(T))
	f.taskNPref = make([]uint32, max1(T))
	f.taskFlags = make([]uint32, max1(T))
	f.taskUIDRank = make([]uint32, max1(T))
	f.taskNzCPU = make([]int64, max1(T))
	f.taskNzMem = make([]int64, max1(T))
	f.taskCtime = make([]int64, max1(T))
	f.taskPrio = make([]int32, max1(T))
	f.taskSelReq = make([]uint64, W*max1(T))
	f.taskTol = make([]uint64, W*max1(T))
	f.taskPortOwn = make([]uint64, W*max1(T))
	f.taskPortConflict = make([]uint64, W*max1(T))
	f.taskAff = make([]uint64, maxAffTerms*W*max1(T))
	f.taskPref = make([]uint64, maxPrefTerms*W*max1(T))
	f.taskPrefWeight = make([]int32, maxPrefTerms*max1(T))
	for ti, t := range f.Tasks {
		pod := t.Pod
		f.taskResPresent[ti] = f.resourceVec(t.Resreq, f.taskResreq, T, ti)
		f.resourceVec(t.InitResreq, f.taskInitreq, T, ti)
		f.taskNzCPU[ti], f.taskNzMem[ti] = podNonzero(pod)
		for _, a := range terms[ti].sel {
			setbit(f.taskSelReq, T, ti, a)
		}
		f.taskNAff[ti] = uint32(len(terms[ti].aff))
		for k, as := range terms[ti].aff {
			for _, a := range as {
				f.taskAff[(k*W+int(a/64))*T+ti] |= uint64(1) << (a % 64)
			}
		}
		f.taskNPref[ti] = uint32(len(terms[ti].pref))
		for k, as := range terms[ti].pref {
			f.taskPrefWeight[k*T+ti] = terms[ti].prefW[k]
			for _, a := range as {
				f.taskPref[(k*W+int(a/64))*T+ti] |= uint64(1) << (a % 64)
			}
		}
		for i := range taintList { // v1helper.TolerationsTolerateTaint (predicates.go:1611)
			if v1helper.TolerationsTolerateTaint(pod.Spec.Tolerations, &taintList[i]) {
				setbit(f.taskTol, T, ti, uint32(i))
			}
		}
		for _, p := range hostPorts(pod) {
			setbit(f.taskPortOwn, T, ti, ports[p])
			for i, other := range portList {
				if portsConflict(p, other) {
					setbit(f.taskPortConflict, T, ti, uint32(i))
				}
			}
		}
		var fl uint32
		if v1qos.GetPodQOS(pod) == v1.PodQOSBestEffort { // predicates.go:1633-1650
			fl |= uint32(C.KB_TASK_BEST_EFFORT_QOS)
		}
		if len(terms[ti].pref) > 0 {
			fl |= uint32(C.KB_TASK_HAS_PREFERRED_NODE_AFFINITY)
		}
		f.taskFlags[ti] = fl
		f.taskPrio[ti] = t.Priority
		f.taskCtime[ti] = pod.CreationTimestamp.UnixNano()
		f.taskUIDRank[ti] = uidRank[string(t.UID)]
	}

	// ---- jobs / queues ----
	f.jobMinAvail = make([]int32, max1(J))
	f.jobReady0 = make([]int32, max1(J))
	f.jobPrio = make([]int32, max1(J))
	f.jobAlloc0 = make([]float64, R*max1(J))
	f.jobAlloc0Present = make([]uint32, max1(J))
	f.jobQueue = make([]uint32, max1(J))
	f.jobCtime = make([]int64, max1(J))
	for j, id := range f.JobIDs {
		job := ssn.Jobs[id]
		f.jobMinAvail[j] = job.MinAvailable
		f.jobReady0[j] = job.ReadyTaskNum() // job_info.go:383
		f.jobPrio[j] = job.Priority
		f.jobCtime[j] = job.CreationTimestamp.UnixNano()
		f.jobQueue[j] = qidx[job.Queue]
		// drf.go:71-77: sum of Resreq over the job's AllocatedStatus tasks (JobInfo.Allocated is that sum, job_info.go:247-264)
		f.jobAlloc0Present[j] = f.resourceVec(job.Allocated, f.jobAlloc0, J, j)
	}
	f.queueWeight = make([]int32, max1(Q))
	f.queueCtime = make([]int64, max1(Q))
	for q, id := range f.QueueIDs {
		qi := ssn.Queues[id]
		f.queueWeight[q] = qi.Weight
		if qi.Queue != nil {
			f.queueCtime[q] = qi.Queue.CreationTimestamp.UnixNano()
		}
	}
	f.buildTiers(ssn.Tiers)
	nidx := make(map[string]int, N)
	for i, name := range f.NodeNames {
		nidx[name] = i
	}
	pa, err := flattenPodAffinity(ssn, f, nidx, &f.snapFlags)
	if err != nil {
		return nil, err
	}
	f.podAff = pa
	return f, nil
}

// buildTiers copies []conf.Tier into C memory (strings, option array, tier array: kb_plugin_conf may only reference C
// memory under the cgo pointer rules): conf.PluginOption -> kb_plugin_option; Enabled* nil -> 0 exactly like the
// framework's isEnabled (session_plugins.go:371) — after plugins.ApplyPluginConfDefaults the *bool fields are non-nil.
func (f *Flat) buildTiers(tiers []conf.Tier) {
	keep := func(p unsafe.Pointer) unsafe.Pointer {
		f.cstrings = append(f.cstrings, (*C.char)(p))
		return p
	}
	cs := func(s string) *C.char { return (*C.char)(keep(unsafe.Pointer(C.CString(s)))) }
	en := func(b *bool) C.uint8_t {
		if b != nil && *b {
			return 1
		}
		return 0
	}
	total := 0
	for _, t := range tiers {
		total += len(t.Plugins)
	}
	f.nTiers = len(tiers)
	optMem := keep(C.calloc(C.size_t(max1(total)), C.size_t(unsafe.Sizeof(C.kb_plugin_option{}))))
	tierMem := keep(C.calloc(C.size_t(max1(len(tiers))), C.size_t(unsafe.Sizeof(C.kb_tier{}))))
	opts := (*[1 << 20]C.kb_plugin_option)(optMem)[:max1(total):max1(total)]
	cts := (*[1 << 20]C.kb_tier)(tierMem)[:max1(len(tiers)):max1(len(tiers))]
	f.cTiers = (*C.kb_tier)(tierMem)
	k := 0
	for ti, t := range tiers {
		cts[ti].n_plugins = C.uint32_t(len(t.Plugins))
		if len(t.Plugins) > 0 {
			cts[ti].plugins = &opts[k]
		}
		for _, p := range t.Plugins {
			o := &opts[k]
			k++
			o.name = cs(p.Name)
			o.enabled_job_order, o.enabled_job_ready, o.enabled_job_pipelined = en(p.EnabledJobOrder), en(p.EnabledJobReady), en(p.EnabledJobPipelined)
			o.enabled_task_order, o.enabled_preemptable, o.enabled_reclaimable = en(p.EnabledTaskOrder), en(p.EnabledPreemptable), en(p.EnabledReclaimable)
			o.enabled_queue_order, o.enabled_predicate, o.enabled_node_order = en(p.EnabledQueueOrder), en(p.EnabledPredicate), en(p.EnabledNodeOrder)
			keys := make([]string, 0, len(p.Arguments))
			for key := range p.Arguments {
				keys = append(keys, key)
			}
			sort.Strings(keys)
			if len(keys) == 0 {
				continue
			}
			psz := C.size_t(unsafe.Sizeof((*C.char)(nil)))
			ka := (*[1 << 20]*C.char)(keep(C.calloc(C.size_t(len(keys)), psz)))
			va := (*[1 << 20]*C.char)(keep(C.calloc(C.size_t(len(keys)), psz)))
			for i, key := range keys {
				ka[i] = cs(key)
				va[i] = cs(p.Arguments[key])
			}
			o.n_args = C.uint32_t(len(keys))
			o.arg_keys = (**C.char)(unsafe.Pointer(ka))
			o.arg_values = (**C.char)(unsafe.Pointer(va))
		}
	}
}

// Free releases the C copy of the tier configuration.
func (f *Flat) Free() {
	for _, p := range f.cstrings {
		C.free(unsafe.Pointer(p))
	}
	f.cstrings = nil
}

// arena holds C copies of the SoA slices for one kb_session_load call.  cgo forbids handing C a struct (kb_snapshot) that
// contains Go pointers, so the arrays are copied into C memory (a few MB per cycle, well under a millisecond) and the
// struct only ever holds C pointers.
type arena struct{ ptrs []unsafe.Pointer }

func (a *arena) put(p unsafe.Pointer, n uintptr) unsafe.Pointer {
	c := C.malloc(C.size_t(n))
	C.memcpy(c, p, C.size_t(n))
	a.ptrs = append(a.ptrs, c)
	return c
}
func (a *arena) free() {
	for _, p := range a.ptrs {
		C.free(p)
	}
	a.ptrs = nil
}
func (a *arena) f64(s []float64) *C.double  { return (*C.double)(a.put(unsafe.Pointer(&s[0]), uintptr(len(s))*8)) }
func (a *arena) u32(s []uint32) *C.uint32_t { return (*C.uint32_t)(a.put(unsafe.Pointer(&s[0]), uintptr(len(s))*4)) }
func (a *arena) i32(s []int32) *C.int32_t   { return (*C.int32_t)(a.put(unsafe.Pointer(&s[0]), uintptr(len(s))*4)) }
func (a *arena) i64(s []int64) *C.int64_t   { return (*C.int64_t)(a.put(unsafe.Pointer(&s[0]), uintptr(len(s))*8)) }
func (a *arena) u64(s []uint64) *C.uint64_t { return (*C.uint64_t)(a.put(unsafe.Pointer(&s[0]), uintptr(len(s))*8)) }

// cSnapshot fills a kb_snapshot whose arrays live in `a` (every slice has >= 1 element).  Engine.Load frees the arena
// after kb_session_load returns: the library copies everything it needs before returning.
func (f *Flat) cSnapshot(s *C.kb_snapshot, a *arena) {
	s.abi_version = C.KB_ABI_VERSION
	s.flags = C.uint32_t(f.snapFlags)
	s.pod_affinity = nil
	if f.podAff != nil {
		s.pod_affinity = f.podAff.cPodAffinity(a)
	}
	s.R, s.W, s.N, s.T, s.J, s.Q = C.uint32_t(f.R), C.uint32_t(f.W), C.uint32_t(f.N), C.uint32_t(f.T), C.uint32_t(f.J), C.uint32_t(f.Q)
	s.node_idle, s.node_releasing, s.node_used, s.node_allocatable = a.f64(f.nodeIdle), a.f64(f.nodeReleasing), a.f64(f.nodeUsed), a.f64(f.nodeAllocatable)
	s.node_alloc_present, s.node_flags = a.u32(f.nodeAllocPresent), a.u32(f.nodeFlags)
	s.node_alloc_cpu, s.node_alloc_mem, s.node_nz_cpu, s.node_nz_mem = a.i64(f.nodeAllocCPU), a.i64(f.nodeAllocMem), a.i64(f.nodeNzCPU), a.i64(f.nodeNzMem)
	s.node_pods, s.node_max_pods = a.i32(f.nodePods), a.i32(f.nodeMaxPods)
	s.node_labels, s.node_taints, s.node_ports = a.u64(f.nodeLabels), a.u64(f.nodeTaints), a.u64(f.nodePorts)
	s.task_initreq, s.task_resreq, s.task_res_present = a.f64(f.taskInitreq), a.f64(f.taskResreq), a.u32(f.taskResPresent)
	s.task_nz_cpu, s.task_nz_mem = a.i64(f.taskNzCPU), a.i64(f.taskNzMem)
	s.task_sel_req, s.task_aff_terms, s.task_n_aff_terms = a.u64(f.taskSelReq), a.u64(f.taskAff), a.u32(f.taskNAff)
	s.task_tol, s.task_port_own, s.task_port_conflict = a.u64(f.taskTol), a.u64(f.taskPortOwn), a.u64(f.taskPortConflict)
	s.task_flags, s.task_prio, s.task_ctime, s.task_uid_rank = a.u32(f.taskFlags), a.i32(f.taskPrio), a.i64(f.taskCtime), a.u32(f.taskUIDRank)
	s.job_task_off, s.job_min_avail, s.job_ready0 = a.u32(f.jobTaskOff), a.i32(f.jobMinAvail), a.i32(f.jobReady0)
	s.job_alloc0, s.job_alloc0_present, s.job_queue = a.f64(f.jobAlloc0), a.u32(f.jobAlloc0Present), a.u32(f.jobQueue)
	s.job_prio, s.job_ctime = a.i32(f.jobPrio), a.i64(f.jobCtime)
	s.queue_weight, s.queue_ctime = a.i32(f.queueWeight), a.i64(f.queueCtime)
	s.task_n_pref_terms, s.task_pref_terms, s.task_pref_weights = a.u32(f.taskNPref), a.u64(f.taskPref), a.i32(f.taskPrefWeight)
}
