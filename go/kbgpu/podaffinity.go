package kbgpu

/*
#include "kbgpu.h"
*/
import "C"

import (
	"encoding/json"
	"fmt"
	"sort"
	"strings"
	"unsafe"

	v1 "k8s.io/api/core/v1"
	metav1 "k8s.io/apimachinery/pkg/apis/meta/v1"
	"k8s.io/apimachinery/pkg/labels"
	"k8s.io/apimachinery/pkg/util/sets"
	priorityutil "k8s.io/kubernetes/pkg/scheduler/algorithm/priorities/util"

	"github.com/kubernetes-sigs/kube-batch/pkg/scheduler/api"
	"github.com/kubernetes-sigs/kube-batch/pkg/scheduler/framework"
)

// podAff is the Go side of kb_pod_affinity (include/kbgpu.h): inter-pod (anti)affinity flattened into counter groups per
// topology domain (predicate step 10) and pod kinds with per-task weight lists (InterPodAffinityPriority).  The executable
// specification is kube_batch_b200/builder.py::flatten_pod_affinity, which tests/test_pod_affinity.py checks against an
// object-level restatement of the vendored predicates.go:1261-1572 / interpod_affinity.go:99-235; this file is the same
// computation over the real objects, with the matching done by the reference's own helpers.  UNVERIFIED BY A COMPILER HERE.
type podAff struct {
	nKeysets, nGroups, nKinds int
	firstUnbound              int32
	nodeDomain                []int32 // [nKeysets][N]
	keysetDomains             []uint32
	groupKeyset               []uint32
	groupCount0, groupTotal0  []int32
	taskForbid, taskContrib   []uint64 // groups 0..63
	taskXgroupOff, taskXgroup []uint32 // groups >= 64: (g << 2) | KB_XGROUP_FORBID | KB_XGROUP_CONTRIB; nil when nGroups <= 64
	taskNeed, taskKind        []int32
	nodeKindCount0            []int32 // [nKinds][N]
	kindUnbound               []uint8
	taskWeightOff             []uint32
	weightKind, weightKeyset  []int32
	weightValue               []int64
	members                   map[*v1.Pod]bool     // listed pods that are members of a counter group: KB_RUNNING_AFF_MEMBER for the Running ones
	memberGroups              map[*v1.Pod][]uint32 // the groups of each listed pod, ascending: kb_running.aff_group for the Running ones
}

// termProps is what a term selects: GetNamespacesFromPodAffinityTerm + LabelSelectorAsSelector (topologies.go:25-49)
type termProps struct {
	ns  sets.String
	sel labels.Selector
	key string // canonical form, for interning
}

func propsOf(owner *v1.Pod, term *v1.PodAffinityTerm) (termProps, error) {
	sel, err := metav1.LabelSelectorAsSelector(term.LabelSelector)
	if err != nil {
		return termProps{}, err
	}
	ns := priorityutil.GetNamespacesFromPodAffinityTerm(owner, term)
	nilSel := "sel"
	if term.LabelSelector == nil {
		nilSel = "nil" // labels.Nothing() and labels.Everything() both print as ""
	}
	return termProps{ns, sel, strings.Join(ns.List(), ",") + "|" + nilSel + "|" + sel.String()}, nil
}

func (p termProps) matches(pod *v1.Pod) bool { return priorityutil.PodMatchesTermsNamespaceAndSelector(pod, p.ns, p.sel) }

func requiredTerms(pod *v1.Pod, anti bool) []v1.PodAffinityTerm {
	a := pod.Spec.Affinity
	if a == nil {
		return nil
	}
	if anti {
		if a.PodAntiAffinity == nil {
			return nil
		}
		return a.PodAntiAffinity.RequiredDuringSchedulingIgnoredDuringExecution
	}
	if a.PodAffinity == nil {
		return nil
	}
	return a.PodAffinity.RequiredDuringSchedulingIgnoredDuringExecution
}

func preferredTerms(pod *v1.Pod, anti bool) []v1.WeightedPodAffinityTerm {
	a := pod.Spec.Affinity
	if a == nil {
		return nil
	}
	if anti {
		if a.PodAntiAffinity == nil {
			return nil
		}
		return a.PodAntiAffinity.PreferredDuringSchedulingIgnoredDuringExecution
	}
	if a.PodAffinity == nil {
		return nil
	}
	return a.PodAffinity.PreferredDuringSchedulingIgnoredDuringExecution
}

func hasPodAffinity(pod *v1.Pod) bool {
	a := pod.Spec.Affinity
	return a != nil && (a.PodAffinity != nil || a.PodAntiAffinity != nil)
}

// podType: pods with the same namespace, labels and (anti)affinity spec are interchangeable for every match below
func podType(pod *v1.Pod) string {
	var aff, anti []byte
	if a := pod.Spec.Affinity; a != nil {
		aff, _ = json.Marshal(a.PodAffinity)
		anti, _ = json.Marshal(a.PodAntiAffinity)
	}
	return pod.Namespace + "\x00" + labels.Set(pod.Labels).String() + "\x00" + string(aff) + "\x00" + string(anti)
}

type placedPod struct {
	pod     *v1.Pod
	node    int
	unbound bool
}

// flattenPodAffinity returns nil when no pod of the session carries inter-pod terms.  snapFlags receives
// KB_SNAPSHOT_PLACED_POD_AFFINITY / KB_SNAPSHOT_LISTED_POD_WITHOUT_NODE.
func flattenPodAffinity(ssn *framework.Session, f *Flat, nidx map[string]int, snapFlags *uint32) (*podAff, error) {
	N, T := len(f.NodeNames), len(f.Tasks)
	// util.PodLister (plugins/util/util.go:37-85): AllocatedStatus tasks of the session's jobs, located by TaskInfo.NodeName
	var listed []placedPod
	any := false
	for _, id := range f.JobIDs {
		job := ssn.Jobs[id]
		for status, tasks := range job.TaskStatusIndex {
			if !api.AllocatedStatus(status) {
				continue
			}
			for _, t := range tasks {
				n, ok := nidx[t.NodeName]
				if !ok { // CachedNodeInfo.GetNodeInfo fails: every InterPodAffinityMatches call of the session errors (kbgpu.h)
					*snapFlags |= C.KB_SNAPSHOT_LISTED_POD_WITHOUT_NODE
					continue
				}
				listed = append(listed, placedPod{t.Pod, n, t.Pod.Spec.NodeName == ""})
				if hasPodAffinity(t.Pod) {
					any = true
					*snapFlags |= C.KB_SNAPSHOT_PLACED_POD_AFFINITY
				}
			}
		}
	}
	// NodeInfo.Tasks of every node, whatever the status: what nodeInfo.Pods() hands the priority
	var inTasks []placedPod
	firstUnbound := int32(-1)
	for n, name := range f.NodeNames {
		for _, t := range ssn.Nodes[name].Tasks {
			unbound := t.Pod.Spec.NodeName == ""
			inTasks = append(inTasks, placedPod{t.Pod, n, unbound})
			if unbound && firstUnbound < 0 {
				firstUnbound = int32(n)
			}
			if hasPodAffinity(t.Pod) {
				any = true
				*snapFlags |= C.KB_SNAPSHOT_PLACED_POD_AFFINITY
			}
		}
	}
	for _, t := range f.Tasks {
		if hasPodAffinity(t.Pod) {
			any = true
		}
	}
	if !any {
		return nil, nil
	}

	// ---- pod types ----
	typeID := map[string]int{}
	var reps []*v1.Pod
	typeOf := func(pod *v1.Pod) int {
		k := podType(pod)
		id, ok := typeID[k]
		if !ok {
			id = len(reps)
			typeID[k] = id
			reps = append(reps, pod)
		}
		return id
	}
	ptype := make([]int, T)
	pendSet := map[int]bool{}
	for i, t := range f.Tasks {
		ptype[i] = typeOf(t.Pod)
		pendSet[ptype[i]] = true
	}
	ltype := make([]int, len(listed))
	for i, p := range listed {
		ltype[i] = typeOf(p.pod)
	}
	ttype := make([]int, len(inTasks))
	for i, p := range inTasks {
		ttype[i] = typeOf(p.pod)
	}
	pendTypes := make([]int, 0, len(pendSet))
	for ty := range pendSet {
		pendTypes = append(pendTypes, ty)
	}
	sort.Ints(pendTypes)

	// ---- key sets and domains ----
	pa := &podAff{firstUnbound: firstUnbound}
	keysetID := map[string]int{}
	keysetOf := func(keys []string) (int, error) {
		ks := append([]string(nil), keys...)
		sort.Strings(ks)
		uniq := ks[:0]
		for i, k := range ks {
			if k == "" {
				return 0, &ErrUnsupported{"a required pod (anti)affinity term with an empty topologyKey (an error in the reference, predicates.go:1311-1313)"}
			}
			if i == 0 || k != ks[i-1] {
				uniq = append(uniq, k)
			}
		}
		id := strings.Join(uniq, "\x00")
		if s, ok := keysetID[id]; ok {
			return s, nil
		}
		s := len(keysetID)
		keysetID[id] = s
		vals := map[string]int32{}
		row := make([]int32, N)
		for n, name := range f.NodeNames {
			node := ssn.Nodes[name].Node
			row[n] = -1
			v := make([]string, 0, len(uniq))
			ok := node != nil
			for _, k := range uniq {
				if !ok {
					break
				}
				lv, has := node.Labels[k]
				ok = ok && has
				v = append(v, lv)
			}
			if ok {
				vk := strings.Join(v, "\x00")
				d, seen := vals[vk]
				if !seen {
					d = int32(len(vals))
					vals[vk] = d
				}
				row[n] = d
			}
		}
		pa.nodeDomain = append(pa.nodeDomain, row...)
		pa.keysetDomains = append(pa.keysetDomains, uint32(len(vals)))
		return s, nil
	}

	// ---- predicate groups ----
	type group struct {
		keyset int
		member []bool // by pod type
	}
	var groups []group
	groupID := map[string]int{}
	addGroup := func(key string, keyset int, member func(*v1.Pod) bool) int {
		if g, ok := groupID[key]; ok {
			return g
		}
		g := len(groups)
		groupID[key] = g
		m := make([]bool, len(reps))
		for ty, rep := range reps {
			m[ty] = member(rep)
		}
		groups = append(groups, group{keyset, m})
		return g
	}
	forbid := map[int]map[int]bool{} // pending type -> the groups it forbids (any number of groups)
	addForbid := func(ty, g int) {
		if forbid[ty] == nil {
			forbid[ty] = map[int]bool{}
		}
		forbid[ty][g] = true
	}
	need := map[int]int32{}
	selfMatch := map[int]bool{}
	for _, ty := range pendTypes {
		need[ty] = -1
	}
	// (A) required anti-affinity terms pods own: satisfiesExistingPodsAntiAffinity (predicates.go:1400-1439)
	ownerSet := map[int]bool{}
	for _, ty := range ltype {
		ownerSet[ty] = true
	}
	for _, ty := range pendTypes {
		ownerSet[ty] = true
	}
	owners := make([]int, 0, len(ownerSet))
	for ty := range ownerSet {
		owners = append(owners, ty)
	}
	sort.Ints(owners)
	for _, oty := range owners {
		owner := reps[oty]
		for i := range requiredTerms(owner, true) {
			term := &requiredTerms(owner, true)[i]
			if term.TopologyKey == "" {
				continue // node.Labels[""] never exists: the term rejects nothing (:1366)
			}
			props, err := propsOf(owner, term)
			if err != nil {
				return nil, &ErrUnsupported{"invalid label selector in a pod anti-affinity term: " + err.Error()}
			}
			var victims []int
			for _, ty := range pendTypes {
				if props.matches(reps[ty]) {
					victims = append(victims, ty)
				}
			}
			if len(victims) == 0 {
				continue
			}
			ks, err := keysetOf([]string{term.TopologyKey})
			if err != nil {
				return nil, err
			}
			topo, pkey := term.TopologyKey, props.key
			g := addGroup("A|"+pkey+"|"+topo, ks, func(x *v1.Pod) bool {
				for j := range requiredTerms(x, true) {
					t := &requiredTerms(x, true)[j]
					if t.TopologyKey != topo {
						continue
					}
					if p, err := propsOf(x, t); err == nil && p.key == pkey {
						return true
					}
				}
				return false
			})
			for _, ty := range victims {
				addForbid(ty, g)
			}
		}
	}
	// (B) the pending pods' own required terms: satisfiesPodsAffinityAntiAffinity, slow path (:1516-1562)
	for _, ty := range pendTypes {
		pod := reps[ty]
		for _, anti := range []bool{false, true} {
			terms := requiredTerms(pod, anti)
			if len(terms) == 0 {
				continue
			}
			var props []termProps
			var keys, pkeys []string
			for i := range terms {
				p, err := propsOf(pod, &terms[i])
				if err != nil {
					return nil, &ErrUnsupported{"invalid label selector in a pod (anti)affinity term: " + err.Error()}
				}
				props = append(props, p)
				pkeys = append(pkeys, p.key)
				keys = append(keys, terms[i].TopologyKey)
			}
			ks, err := keysetOf(keys)
			if err != nil {
				return nil, err
			}
			sort.Strings(pkeys)
			all := func(x *v1.Pod) bool { // podMatchesAllAffinityTermProperties (metadata.go:601-612)
				for _, p := range props {
					if !p.matches(x) {
						return false
					}
				}
				return true
			}
			g := addGroup(fmt.Sprintf("B|%s|%d", strings.Join(pkeys, "\x01"), ks), ks, all)
			if anti {
				addForbid(ty, g)
			} else {
				need[ty] = int32(g)
				selfMatch[ty] = all(pod) // targetPodMatchesAffinityOfPod(pod, pod)
			}
		}
	}
	if len(groups) > int(C.KB_MAX_AFF_GROUPS) {
		return nil, &ErrUnsupported{fmt.Sprintf("%d inter-pod affinity counter groups: more than %d", len(groups), int(C.KB_MAX_AFF_GROUPS))}
	}
	if len(keysetID) > 64 {
		return nil, &ErrUnsupported{fmt.Sprintf("%d topology key sets: more than 64", len(keysetID))}
	}
	pa.nGroups = len(groups)
	gOff := make([]int, len(groups)+1)
	for g, gr := range groups {
		pa.groupKeyset = append(pa.groupKeyset, uint32(gr.keyset))
		gOff[g+1] = gOff[g] + int(pa.keysetDomains[gr.keyset])
	}
	pa.groupCount0 = make([]int32, max1(gOff[len(groups)]))
	pa.groupTotal0 = make([]int32, max1(len(groups)))
	pa.members = map[*v1.Pod]bool{}
	pa.memberGroups = map[*v1.Pod][]uint32{}
	for i, p := range listed {
		for g, gr := range groups {
			if !gr.member[ltype[i]] {
				continue
			}
			pa.members[p.pod] = true
			pa.memberGroups[p.pod] = append(pa.memberGroups[p.pod], uint32(g))
			pa.groupTotal0[g]++
			if d := pa.nodeDomain[gr.keyset*N+p.node]; d >= 0 {
				pa.groupCount0[gOff[g]+int(d)]++
			}
		}
	}

	// ---- priority: weights between pod types (processPod, interpod_affinity.go:119-171), kinds, per-task lists ----
	weights := func(in, ex *v1.Pod) map[string]int64 {
		w := map[string]int64{}
		add := func(owner *v1.Pod, term *v1.PodAffinityTerm, check *v1.Pod, v int64) {
			if term.TopologyKey == "" || v == 0 { // NodesHaveSameTopologyKey is false for an empty key
				return
			}
			if p, err := propsOf(owner, term); err == nil && p.matches(check) {
				w[term.TopologyKey] += v
			}
		}
		for i := range preferredTerms(in, false) {
			t := &preferredTerms(in, false)[i]
			add(in, &t.PodAffinityTerm, ex, int64(t.Weight))
		}
		for i := range preferredTerms(in, true) {
			t := &preferredTerms(in, true)[i]
			add(in, &t.PodAffinityTerm, ex, -int64(t.Weight))
		}
		for i := range requiredTerms(ex, false) { // hardPodAffinityWeight = v1.DefaultHardPodAffinitySymmetricWeight (nodeorder.go:159)
			add(ex, &requiredTerms(ex, false)[i], in, int64(v1.DefaultHardPodAffinitySymmetricWeight))
		}
		for i := range preferredTerms(ex, false) {
			t := &preferredTerms(ex, false)[i]
			add(ex, &t.PodAffinityTerm, in, int64(t.Weight))
		}
		for i := range preferredTerms(ex, true) {
			t := &preferredTerms(ex, true)[i]
			add(ex, &t.PodAffinityTerm, in, -int64(t.Weight))
		}
		for k, v := range w {
			if v == 0 {
				delete(w, k)
			}
		}
		return w
	}
	wtab := map[[2]int]map[string]int64{}
	for _, pt := range pendTypes {
		for xt := range reps {
			wtab[[2]int{pt, xt}] = weights(reps[pt], reps[xt])
		}
	}
	kindID := map[string]int{}
	kindRep := map[int]int{}
	kindOf := func(xt int, unbound bool) int32 {
		var sb strings.Builder
		nonzero := false
		for _, pt := range pendTypes {
			w := wtab[[2]int{pt, xt}]
			keys := make([]string, 0, len(w))
			for k := range w {
				keys = append(keys, k)
			}
			sort.Strings(keys)
			for _, k := range keys {
				fmt.Fprintf(&sb, "%s=%d,", k, w[k])
				nonzero = true
			}
			sb.WriteByte(';')
		}
		if !nonzero {
			return -1
		}
		fmt.Fprintf(&sb, "|%v", unbound)
		id, ok := kindID[sb.String()]
		if !ok {
			id = len(kindID)
			kindID[sb.String()] = id
			kindRep[id] = xt
			if unbound {
				pa.kindUnbound = append(pa.kindUnbound, 1)
			} else {
				pa.kindUnbound = append(pa.kindUnbound, 0)
			}
		}
		return int32(id)
	}
	xkind := make([]int32, len(inTasks))
	for i, p := range inTasks {
		xkind[i] = kindOf(ttype[i], p.unbound)
	}
	pkind := map[int]int32{}
	for _, ty := range pendTypes {
		pkind[ty] = kindOf(ty, true) // a task placed in this session keeps an empty Spec.NodeName
	}
	pa.nKinds = len(kindID)
	pa.nodeKindCount0 = make([]int32, max1(pa.nKinds)*max1(N))
	for i, p := range inTasks {
		if xkind[i] >= 0 {
			pa.nodeKindCount0[int(xkind[i])*N+p.node]++
		}
	}
	type wEntry struct {
		kind, keyset int32
		value        int64
	}
	wlist := map[int][]wEntry{}
	for _, pt := range pendTypes {
		for k := 0; k < pa.nKinds; k++ {
			w := wtab[[2]int{pt, kindRep[k]}]
			keys := make([]string, 0, len(w))
			for key := range w {
				keys = append(keys, key)
			}
			sort.Strings(keys)
			for _, key := range keys {
				ks, err := keysetOf([]string{key})
				if err != nil {
					return nil, err
				}
				wlist[pt] = append(wlist[pt], wEntry{int32(k), int32(ks), w[key]})
			}
		}
	}
	if len(keysetID) > 64 {
		return nil, &ErrUnsupported{"more than 64 topology key sets"}
	}
	pa.nKeysets = len(keysetID)

	// ---- per task ----
	pa.taskForbid, pa.taskContrib = make([]uint64, max1(T)), make([]uint64, max1(T))
	pa.taskNeed, pa.taskKind = make([]int32, max1(T)), make([]int32, max1(T))
	pa.taskWeightOff = make([]uint32, T+1)
	if len(groups) > 64 {
		pa.taskXgroupOff = make([]uint32, T+1)
	}
	for t := 0; t < T; t++ {
		ty := ptype[t]
		pa.taskNeed[t] = need[ty]
		pa.taskKind[t] = pkind[ty]
		for g, gr := range groups { // groups < 64: bits of the masks; the others: entries of task_xgroup, ascending
			f, c := forbid[ty][g], gr.member[ty]
			if g < 64 {
				if f {
					pa.taskForbid[t] |= 1 << uint(g)
				}
				if c {
					pa.taskContrib[t] |= 1 << uint(g)
				}
				continue
			}
			if f || c {
				e := uint32(g) << 2
				if f {
					e |= C.KB_XGROUP_FORBID
				}
				if c {
					e |= C.KB_XGROUP_CONTRIB
				}
				pa.taskXgroup = append(pa.taskXgroup, e)
			}
		}
		if pa.taskXgroupOff != nil {
			pa.taskXgroupOff[t+1] = uint32(len(pa.taskXgroup))
		}
		for _, e := range wlist[ty] {
			pa.weightKind = append(pa.weightKind, e.kind)
			pa.weightKeyset = append(pa.weightKeyset, e.keyset)
			pa.weightValue = append(pa.weightValue, e.value)
		}
		pa.taskWeightOff[t+1] = uint32(len(pa.weightKind))
		if hasPodAffinity(f.Tasks[t].Pod) {
			f.taskFlags[t] |= C.KB_TASK_HAS_POD_AFFINITY
		}
		if selfMatch[ty] {
			f.taskFlags[t] |= C.KB_TASK_AFF_SELF_MATCH
		}
	}
	return pa, nil
}

// cPodAffinity copies the tables into the arena and returns the C struct (itself in C memory: kb_snapshot may only hold C pointers)
func (pa *podAff) cPodAffinity(a *arena) *C.kb_pod_affinity {
	one32, one64, oneU := []int32{0}, []int64{0}, []uint32{0}
	i32 := func(s []int32) *C.int32_t {
		if len(s) == 0 {
			s = one32
		}
		return a.i32(s)
	}
	u32 := func(s []uint32) *C.uint32_t {
		if len(s) == 0 {
			s = oneU
		}
		return a.u32(s)
	}
	i64 := func(s []int64) *C.int64_t {
		if len(s) == 0 {
			s = one64
		}
		return a.i64(s)
	}
	var c C.kb_pod_affinity
	c.n_keysets, c.n_groups, c.n_kinds = C.uint32_t(pa.nKeysets), C.uint32_t(pa.nGroups), C.uint32_t(pa.nKinds)
	c.n_weights = C.uint32_t(len(pa.weightKind))
	c.first_unbound_node = C.int32_t(pa.firstUnbound)
	c.node_domain, c.keyset_domains, c.group_keyset = i32(pa.nodeDomain), u32(pa.keysetDomains), u32(pa.groupKeyset)
	c.group_count0, c.group_total0 = i32(pa.groupCount0), i32(pa.groupTotal0)
	c.task_forbid, c.task_contrib = a.u64(pa.taskForbid), a.u64(pa.taskContrib)
	c.task_need, c.task_kind = i32(pa.taskNeed), i32(pa.taskKind)
	c.node_kind_count0 = i32(pa.nodeKindCount0)
	ku := pa.kindUnbound
	if len(ku) == 0 {
		ku = []uint8{0}
	}
	c.kind_unbound = (*C.uint8_t)(a.put(unsafe.Pointer(&ku[0]), uintptr(len(ku))))
	c.task_weight_off = u32(pa.taskWeightOff)
	c.weight_kind, c.weight_keyset, c.weight_value = i32(pa.weightKind), i32(pa.weightKeyset), i64(pa.weightValue)
	if pa.taskXgroupOff != nil { // NULL for sessions with at most 64 groups
		c.task_xgroup_off, c.task_xgroup = u32(pa.taskXgroupOff), u32(pa.taskXgroup)
	}
	return (*C.kb_pod_affinity)(a.put(unsafe.Pointer(&c), unsafe.Sizeof(c)))
}
