"""Object-level session builder -> flattened Snapshot (the "flattener").

Mirrors the in-memory harness of the reference's action tests
(kube-batch/pkg/scheduler/actions/allocate/allocate_test.go:150-198: objects are fed through
cache.AddNode / AddPod / AddPodGroup / AddQueue, then framework.OpenSession takes cache.Snapshot())
and the helper constructors of kube-batch/pkg/scheduler/util/test_utils.go:34-93.  It is also the
executable specification of what the Go shim's flattening must compute (INTEGRATION.md):

  * canonical orders: nodes by Name, jobs by JobID "<ns>/<podgroup>", queues by QueueID (= Name),
    task_uid_rank = rank of Pod.UID;
  * selector / required-affinity requirements, NoSchedule|NoExecute taints and host ports are
    interned per snapshot into bit "atoms";
  * node aggregates (Idle / Used / Releasing, pod count, non-zero request sums, used ports) follow
    api.NodeInfo.AddTask (api/node_info.go:172-212) and k8s nodeinfo.AddPod
    (vendor/k8s.io/kubernetes/pkg/scheduler/nodeinfo/node_info.go:502-524).
"""
from __future__ import annotations

import math

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import abi
from .snapshot import Snapshot

DEFAULT_MILLI_CPU_REQUEST = 100                 # priorities/util/non_zero.go:36
DEFAULT_MEMORY_REQUEST = 200 * 1024 * 1024      # :38
GPU = "nvidia.com/gpu"

_SUFFIX = {"Ki": 1 << 10, "Mi": 1 << 20, "Gi": 1 << 30, "Ti": 1 << 40,
           "k": 10 ** 3, "M": 10 ** 6, "G": 10 ** 9, "T": 10 ** 12}


def parse_quantity(q) -> float:
    """resource.MustParse for the forms the reference tests use ("1", "500m", "4Gi", "1G")."""
    if isinstance(q, (int, float)):
        return float(q)
    s = str(q)
    if s.endswith("m"):
        return float(s[:-1]) / 1000.0
    for suf in ("Ki", "Mi", "Gi", "Ti", "k", "M", "G", "T"):
        if s.endswith(suf):
            return float(s[: -len(suf)]) * _SUFFIX[suf]
    return float(s)


def build_resource_list(cpu, memory, gpu="0") -> Dict[str, float]:
    """util.BuildResourceList / BuildResourceListWithGPU (util/test_utils.go:34-49):
    cpu in cores, memory in bytes, nvidia.com/gpu always present."""
    return {"cpu": parse_quantity(cpu), "memory": parse_quantity(memory), GPU: parse_quantity(gpu)}


@dataclass
class Node:
    name: str
    allocatable: Dict[str, float]                 # ResourceList: cpu (cores), memory (bytes), pods, scalars (units)
    labels: Dict[str, str] = field(default_factory=dict)
    taints: List[Tuple[str, str, str]] = field(default_factory=list)   # (key, value, effect)
    unschedulable: bool = False
    ready: Optional[bool] = None                  # NodeReady condition status; None = condition absent
    network_unavailable: Optional[bool] = None
    memory_pressure: bool = False
    disk_pressure: bool = False
    pid_pressure: bool = False


@dataclass
class PodAffinityTerm:
    """v1.PodAffinityTerm: labelSelector (matchLabels + matchExpressions; nil_selector = the Go nil *LabelSelector, which
    LabelSelectorAsSelector turns into labels.Nothing()), namespaces (empty = the owning pod's namespace), topologyKey."""
    topology_key: str
    match_labels: Dict[str, str] = field(default_factory=dict)
    match_expressions: List[Tuple[str, str, Sequence[str]]] = field(default_factory=list)   # In NotIn Exists DoesNotExist
    namespaces: List[str] = field(default_factory=list)
    nil_selector: bool = False


@dataclass
class PodAffinity:
    """v1.PodAffinity / v1.PodAntiAffinity: requiredDuringSchedulingIgnoredDuringExecution and
    preferredDuringSchedulingIgnoredDuringExecution [(weight, term)]."""
    required: List[PodAffinityTerm] = field(default_factory=list)
    preferred: List[Tuple[int, PodAffinityTerm]] = field(default_factory=list)


@dataclass
class Pod:
    namespace: str
    name: str
    node_name: str = ""
    phase: str = "Pending"                        # Pending | Running | Succeeded | Failed | Unknown
    requests: Dict[str, float] = field(default_factory=dict)   # single container; keys may be absent
    init_requests: List[Dict[str, float]] = field(default_factory=list)
    group: str = ""
    labels: Dict[str, str] = field(default_factory=dict)
    node_selector: Dict[str, str] = field(default_factory=dict)
    # required node affinity: OR over terms, each an AND of (key, op, values), op in In NotIn Exists DoesNotExist Gt Lt
    affinity_terms: Optional[List[List[Tuple[str, str, Sequence[str]]]]] = None
    # nodeAffinity.preferredDuringSchedulingIgnoredDuringExecution: [(weight, [(key, op, values), ...]), ...]
    preferred_terms: List[Tuple[int, List[Tuple[str, str, Sequence[str]]]]] = field(default_factory=list)
    tolerations: List[Tuple[str, str, str, str]] = field(default_factory=list)   # (key, operator, value, effect)
    host_ports: List[Tuple[str, str, int]] = field(default_factory=list)          # (hostIP, protocol, hostPort)
    priority: Optional[int] = None
    creation: int = 0
    deleting: bool = False
    uid: Optional[str] = None
    limits: Dict[str, float] = field(default_factory=dict)
    pod_affinity: Optional[PodAffinity] = None          # Spec.Affinity.PodAffinity (None = nil)
    pod_anti_affinity: Optional[PodAffinity] = None     # Spec.Affinity.PodAntiAffinity


@dataclass
class PodGroup:
    namespace: str
    name: str
    queue: str
    min_member: int = 0
    priority: int = 0                             # resolved PriorityClass value (cache.go:664-674)
    creation: int = 0


@dataclass
class Queue:
    name: str
    weight: int = 1
    creation: int = 0


def build_node(name, alloc: Dict[str, float], labels=None, pods: Optional[int] = None) -> Node:
    """util.BuildNode (util/test_utils.go:52-63).  NB the reference helper sets no `pods` capacity, so
    MaxTaskNum = 0 and the predicates plugin rejects every such node (predicates.go:127)."""
    a = dict(alloc)
    if pods is not None:
        a["pods"] = pods
    return Node(name, a, dict(labels or {}))


def build_pod(namespace, name, nodename, phase, req, group_name, labels=None, selector=None) -> Pod:
    """util.BuildPod (util/test_utils.go:66-93)."""
    return Pod(namespace, name, nodename, phase, dict(req), group=group_name, labels=dict(labels or {}),
               node_selector=dict(selector or {}), uid=f"{namespace}-{name}")


def _match_requirement(labels: Dict[str, str], key: str, op: str, values: Sequence[str]) -> bool:
    """labels.Requirement.Matches via v1helper.NodeSelectorRequirementsAsSelector
    (vendor/k8s.io/kubernetes/pkg/apis/core/v1/helper/helpers.go:205-316)."""
    if op == "In":
        return key in labels and labels[key] in values
    if op == "NotIn":
        return key not in labels or labels[key] not in values
    if op == "Exists":
        return key in labels
    if op == "DoesNotExist":
        return key not in labels
    if op in ("Gt", "Lt"):
        if key not in labels:
            return False
        try:
            lv, rv = int(labels[key]), int(values[0])
        except (ValueError, IndexError):
            return False
        return lv > rv if op == "Gt" else lv < rv
    raise ValueError(f"unknown operator {op}")


def _tolerates(tol: Tuple[str, str, str, str], taint: Tuple[str, str, str]) -> bool:
    """Toleration.ToleratesTaint (vendor/k8s.io/api/core/v1/toleration.go:37-56)."""
    key, op, value, effect = tol
    tkey, tvalue, teffect = taint
    if effect and effect != teffect:
        return False
    if key and key != tkey:
        return False
    if op in ("", "Equal"):
        return value == tvalue
    if op == "Exists":
        return True
    return False


def _sanitize_port(ip: str, proto: str, port: int):
    return (ip or "0.0.0.0", proto or "TCP", int(port))   # HostPortInfo.sanitize (host_ports.go:127-135)


def _ports_conflict(a, b) -> bool:
    """HostPortInfo.CheckConflict (host_ports.go:96-125): same (proto, port) and equal IPs or a wildcard."""
    if a[1] != b[1] or a[2] != b[2]:
        return False
    return a[0] == b[0] or a[0] == "0.0.0.0" or b[0] == "0.0.0.0"


class SessionBuilder:
    def __init__(self):
        self.nodes: List[Node] = []
        self.pods: List[Pod] = []
        self.pod_groups: List[PodGroup] = []
        self.queues: List[Queue] = []

    def add_node(self, n: Node):
        self.nodes.append(n)
        return self

    def add_pod(self, p: Pod):
        self.pods.append(p)
        return self

    def add_pod_group(self, g: PodGroup):
        self.pod_groups.append(g)
        return self

    def add_queue(self, q: Queue):
        self.queues.append(q)
        return self

    # ---- api.NewResource (api/resource_info.go:73-90): cpu -> milli, memory -> bytes, scalars -> milli ----
    @staticmethod
    def _milli(q: float) -> int:
        """resource.Quantity.MilliValue(): rounds UP (apimachinery resource/quantity.go ScaledValue), e.g. cpu 0.0005 -> 1."""
        return int(math.ceil(q * 1000.0 - 1e-9))

    @staticmethod
    def _resource(rl: Dict[str, float], dims: List[str]):
        v = np.zeros(len(dims))
        present = 0
        for k, q in rl.items():
            if k == "cpu":
                v[0] += SessionBuilder._milli(q)
            elif k == "memory":
                v[1] += q
            elif k == "pods":
                continue
            else:
                r = dims.index(k)
                v[r] += SessionBuilder._milli(q)
                present |= 1 << r
        return v, present

    @staticmethod
    def _less_equal(l, lpresent: int, r, rpresent: int) -> bool:
        """Resource.LessEqual (resource_info.go:268-302) on dense vectors + scalar-presence masks."""
        def le(a, b, diff):
            return a < b or abs(a - b) < diff
        if not le(l[0], r[0], 10.0) or not le(l[1], r[1], 10.0 * 1024 * 1024):
            return False
        for k in range(2, len(l)):
            if not (lpresent >> k) & 1 or l[k] <= 10.0:
                continue
            if (rpresent >> 2) == 0:
                return False
            if not le(l[k], r[k] if (rpresent >> k) & 1 else 0.0, 10.0):
                return False
        return True

    @staticmethod
    def _task_status(p: Pod) -> str:
        """api.getTaskStatus (api/helpers.go:38-62)."""
        if p.phase == "Running":
            return "Releasing" if p.deleting else "Running"
        if p.phase == "Pending":
            if p.deleting:
                return "Releasing"
            return "Pending" if not p.node_name else "Bound"
        return {"Succeeded": "Succeeded", "Failed": "Failed"}.get(p.phase, "Unknown")

    def flatten(self, W: int = 1) -> Snapshot:
        nodes = sorted(self.nodes, key=lambda n: n.name)
        queues = sorted(self.queues, key=lambda q: q.name)
        qidx = {q.name: i for i, q in enumerate(queues)}
        groups = sorted(self.pod_groups, key=lambda g: f"{g.namespace}/{g.name}")
        # cache.Snapshot drops jobs whose queue does not exist (cache/cache.go:652-656)
        groups = [g for g in groups if g.queue in qidx]
        jidx = {f"{g.namespace}/{g.name}": i for i, g in enumerate(groups)}
        nidx = {n.name: i for i, n in enumerate(nodes)}

        scalars = sorted({k for n in nodes for k in n.allocatable if k not in ("cpu", "memory", "pods")} |
                         {k for p in self.pods for rl in [p.requests] + p.init_requests for k in rl if k not in ("cpu", "memory")})
        dims = ["cpu", "memory"] + scalars
        R = max(2, len(dims))
        assert R <= abi.KB_MAX_R

        pending = [p for p in self.pods if self._task_status(p) == "Pending" and f"{p.namespace}/{p.group}" in jidx]
        uids = sorted((p.uid or f"{p.namespace}-{p.name}") for p in pending)
        uid_rank = {u: i for i, u in enumerate(uids)}
        assert len(uid_rank) == len(pending), "duplicate pod UIDs"
        pending.sort(key=lambda p: jidx[f"{p.namespace}/{p.group}"])

        # ---- atoms ----
        req_atoms: Dict[Tuple, int] = {}

        def atom_of(key, op, values):
            k = (key, op, tuple(values))
            if k not in req_atoms:
                req_atoms[k] = len(req_atoms)
            return req_atoms[k]

        for p in pending:
            for k, v in p.node_selector.items():
                atom_of(k, "In", [v])
            for term in (p.affinity_terms or []):
                for (k, op, vals) in term:
                    atom_of(k, op, vals)
            for (_, exprs) in p.preferred_terms:
                for (k, op, vals) in exprs:
                    atom_of(k, op, vals)
        taint_atoms: Dict[Tuple, int] = {}
        for n in nodes:
            for t in n.taints:
                if t[2] in ("NoSchedule", "NoExecute") and t not in taint_atoms:
                    taint_atoms[t] = len(taint_atoms)
        port_atoms: Dict[Tuple, int] = {}
        for p in self.pods:
            for hp in p.host_ports:
                if hp[2] <= 0:
                    continue
                sp = _sanitize_port(*hp)
                if sp not in port_atoms:
                    port_atoms[sp] = len(port_atoms)
        need = max(len(req_atoms), len(taint_atoms), len(port_atoms), 1)
        W = max(W, (need + 63) // 64)
        assert W <= abi.KB_MAX_W, f"{need} label / taint / port atoms > 64 x KB_MAX_W ({abi.KB_MAX_W})"
        assert R <= abi.KB_NARROW_R or W <= abi.KB_NARROW_W, \
            f"{R} resource dimensions > KB_NARROW_R ({abi.KB_NARROW_R}) with {need} atoms > 64 x KB_NARROW_W ({abi.KB_NARROW_W})"

        s = Snapshot(R, W, len(nodes), len(pending), len(groups), len(queues))

        def setbit(arr, w_major_index, atom):
            arr[atom // 64, w_major_index] |= np.uint64(1) << np.uint64(atom % 64)

        # ---- nodes ----
        for i, n in enumerate(nodes):
            v, present = self._resource(n.allocatable, dims)
            s.node_allocatable[:, i] = v
            s.node_idle[:, i] = v
            s.node_alloc_present[i] = present
            s.node_alloc_cpu[i] = int(v[0])
            s.node_alloc_mem[i] = int(v[1])
            s.node_max_pods[i] = int(n.allocatable.get("pods", 0))
            f = 0
            if n.ready is not None and not n.ready:
                f |= abi.KB_NODE_NOT_READY
            if n.network_unavailable is not None and n.network_unavailable:
                f |= abi.KB_NODE_NET_UNAVAILABLE
            if n.unschedulable:
                f |= abi.KB_NODE_UNSCHEDULABLE
            if n.memory_pressure:
                f |= abi.KB_NODE_MEM_PRESSURE
            if n.disk_pressure:
                f |= abi.KB_NODE_DISK_PRESSURE
            if n.pid_pressure:
                f |= abi.KB_NODE_PID_PRESSURE
            s.node_flags[i] = f
            for (k, op, vals), a in req_atoms.items():
                if _match_requirement(n.labels, k, op, vals):
                    setbit(s.node_labels, i, a)
            for t in n.taints:
                if t in taint_atoms:
                    setbit(s.node_taints, i, taint_atoms[t])

        # ---- pods already on nodes / counted in jobs ----
        def pod_resreq(p: Pod):
            return self._resource(p.requests, dims)

        def pod_nz(p: Pod):
            cpu = self._milli(p.requests["cpu"]) if "cpu" in p.requests else DEFAULT_MILLI_CPU_REQUEST
            mem = int(p.requests["memory"]) if "memory" in p.requests else DEFAULT_MEMORY_REQUEST
            return int(cpu), int(mem)

        on_node = set()                     # pods node.AddTask accepted
        for p in self.pods:
            st = self._task_status(p)
            key = f"{p.namespace}/{p.group}"
            v, present = pod_resreq(p)
            if st != "Pending" and key in jidx:
                j = jidx[key]
                if st in ("Bound", "Binding", "Running", "Allocated"):
                    s.job_alloc0[:, j] += v
                    s.job_alloc0_present[j] |= present
                    s.job_ready0[j] += 1
                elif st == "Succeeded":
                    s.job_ready0[j] += 1
            if p.node_name and p.node_name not in nidx and key in jidx and st in ("Bound", "Binding", "Running", "Allocated"):
                # the job lists the task, its node is not part of the session (cache.Snapshot drops NotReady nodes, cache.go:633-640):
                # util.PodLister + CachedNodeInfo.GetNodeInfo make every InterPodAffinityMatches call fail (kbgpu.h)
                s.flags = int(getattr(s, "flags", 0)) | abi.KB_SNAPSHOT_LISTED_POD_WITHOUT_NODE
            if p.node_name and p.node_name in nidx and st != "Pending":
                i = nidx[p.node_name]
                # cache.addTask: the job has the task (above); node.AddTask refuses what does not fit into Idle
                # (allocateIdleResource, node_info.go:161-167), so a snapshot never carries an over-committed node
                if st != "Pipelined" and not self._less_equal(v, present, s.node_idle[:, i], int(s.node_alloc_present[i])):
                    continue
                on_node.add(id(p))
                # api.NodeInfo.AddTask (node_info.go:172-212)
                if st == "Releasing":
                    s.node_idle[:, i] -= v
                    s.node_releasing[:, i] += v
                elif st == "Pipelined":
                    s.node_releasing[:, i] -= v
                else:
                    s.node_idle[:, i] -= v
                s.node_used[:, i] += v
                s.node_pods[i] += 1
                c, m = pod_nz(p)
                s.node_nz_cpu[i] += c
                s.node_nz_mem[i] += m
                for hp in p.host_ports:
                    if hp[2] > 0:
                        setbit(s.node_ports, i, port_atoms[_sanitize_port(*hp)])

        # ---- jobs / queues ----
        for j, g in enumerate(groups):
            s.job_min_avail[j] = g.min_member
            s.job_queue[j] = qidx[g.queue]
            s.job_prio[j] = g.priority
            s.job_ctime[j] = g.creation
        for q, qu in enumerate(queues):
            s.queue_weight[q] = qu.weight
            s.queue_ctime[q] = qu.creation

        # ---- pending tasks ----
        counts = np.zeros(len(groups) + 1, dtype=np.int64)
        for t, p in enumerate(pending):
            j = jidx[f"{p.namespace}/{p.group}"]
            counts[j + 1] += 1
            v, present = pod_resreq(p)
            s.task_resreq[:, t] = v
            s.task_res_present[t] = present
            init = v.copy()
            for rl in p.init_requests:          # api.GetPodResourceRequest (api/pod_info.go:53-73)
                iv, _ = self._resource(rl, dims)
                init = np.maximum(init, iv)
            s.task_initreq[:, t] = init
            c, m = pod_nz(p)
            s.task_nz_cpu[t], s.task_nz_mem[t] = c, m
            for k, val in p.node_selector.items():
                setbit(s.task_sel_req, t, atom_of(k, "In", [val]))
            terms = p.affinity_terms
            if terms is not None:
                assert 0 < len(terms) <= abi.KB_MAX_AFF_TERMS, "collapse the selector into one atom (DESIGN.md)"
                s.task_n_aff_terms[t] = len(terms)
                for ti, term in enumerate(terms):
                    for (k, op, vals) in term:
                        a = atom_of(k, op, vals)
                        s.task_aff_terms[ti, a // 64, t] |= np.uint64(1) << np.uint64(a % 64)
            for taint, a in taint_atoms.items():
                if any(_tolerates(tol, taint) for tol in p.tolerations):
                    setbit(s.task_tol, t, a)
            for hp in p.host_ports:
                if hp[2] <= 0:
                    continue
                sp = _sanitize_port(*hp)
                setbit(s.task_port_own, t, port_atoms[sp])
                for other, a in port_atoms.items():
                    if _ports_conflict(sp, other):
                        setbit(s.task_port_conflict, t, a)
            fl = 0
            if not p.requests and not p.limits:
                fl |= abi.KB_TASK_BEST_EFFORT_QOS
            if p.preferred_terms:                # NodeAffinityPriority (node_affinity.go:34-77); an empty expression list matches every node
                assert len(p.preferred_terms) <= abi.KB_MAX_PREF_TERMS
                fl |= abi.KB_TASK_HAS_PREFERRED_NODE_AFFINITY
                s.task_n_pref_terms[t] = len(p.preferred_terms)
                for pi, (weight, exprs) in enumerate(p.preferred_terms):
                    s.task_pref_weights[pi, t] = weight
                    for (k, op, vals) in exprs:
                        a = atom_of(k, op, vals)
                        s.task_pref_terms[pi, a // 64, t] |= np.uint64(1) << np.uint64(a % 64)
            s.task_flags[t] = fl
            s.task_prio[t] = 1 if p.priority is None else p.priority    # api.NewTaskInfo (job_info.go:82-90)
            s.task_ctime[t] = p.creation
            s.task_uid_rank[t] = uid_rank[p.uid or f"{p.namespace}-{p.name}"]
        s.job_task_off[:] = np.cumsum(counts).astype(np.uint32)
        # ---- Running tasks one by one: what reclaim / preempt walk (node.Tasks); not part of kb_snapshot yet ----
        running = [p for p in self.pods if self._task_status(p) == "Running" and f"{p.namespace}/{p.group}" in jidx and id(p) in on_node]
        ruids = sorted((p.uid or f"{p.namespace}-{p.name}") for p in running)
        rrank = {u: i for i, u in enumerate(ruids)}
        rt = {"node": np.array([nidx[p.node_name] for p in running], dtype=np.uint32),
              "job": np.array([jidx[f"{p.namespace}/{p.group}"] for p in running], dtype=np.uint32),
              "resreq": np.zeros((R, len(running))), "res_present": np.zeros(len(running), dtype=np.uint32),
              "prio": np.array([1 if p.priority is None else p.priority for p in running], dtype=np.int32),
              "ctime": np.array([p.creation for p in running], dtype=np.int64),
              "uid_rank": np.array([rrank[p.uid or f"{p.namespace}-{p.name}"] for p in running], dtype=np.uint32),
              "flags": np.array([1 if (p.namespace == "kube-system" or p.labels.get("priorityClassName") in
                                       ("system-cluster-critical", "system-node-critical")) else 0 for p in running], dtype=np.uint32),
              "names": [f"{p.namespace}/{p.name}" for p in running]}
        for i, p in enumerate(running):
            v, present = pod_resreq(p)
            rt["resreq"][:, i] = v
            rt["res_present"][i] = present
        pod_objects = None
        groups_of = {}
        if any(p.pod_affinity is not None or p.pod_anti_affinity is not None for p in self.pods):
            pend_ids = set(id(p) for p in pending)
            existing = [p for p in self.pods if id(p) not in pend_ids and p.node_name in nidx and self._task_status(p) != "Pending"]
            s.pod_affinity, pod_objects = flatten_pod_affinity(nodes, pending, existing, s, on_node,
                                                               lambda p: self._task_status(p), lambda p: f"{p.namespace}/{p.group}" in jidx)
            members = s.pod_affinity.pop("member_pod_ids")
            groups_of = s.pod_affinity.pop("member_groups")
            for i, p in enumerate(running):
                if id(p) in members:
                    rt["flags"][i] |= abi.KB_RUNNING_AFF_MEMBER      # its eviction would take it out of util.PodLister (kbgpu.h)
        # the counter groups of every Running task (kb_running.aff_group_off / aff_group): kept apart from "running", whose callers
        # without them keep the withholding rule of KB_RUNNING_AFF_MEMBER; merge them in to have the member bits kept exact
        rg = [groups_of.get(id(p), []) for p in running]
        rag = {"aff_group_off": np.concatenate([[0], np.cumsum([len(x) for x in rg], dtype=np.int64)]).astype(np.uint32),
               "aff_group": np.array([g for x in rg for g in x], dtype=np.uint32)}
        s.meta = {"pod_objects": pod_objects, "running": rt, "running_aff_groups": rag, "nodes": [n.name for n in nodes],
                  "tasks": [f"{p.namespace}/{p.name}" for p in pending], "jobs": list(jidx.keys()), "queues": [q.name for q in queues], "dims": dims}
        s.validate()
        return s


# ----------------------------------------------------------------------------------------------
# inter-pod (anti)affinity: the string work of predicate step 10 and InterPodAffinityPriority, done once per snapshot
# (include/kbgpu.h kb_pod_affinity).  Reference: vendor/k8s.io/kubernetes/pkg/scheduler/algorithm/predicates/predicates.go:
# 1261-1572, .../priorities/interpod_affinity.go:99-235, .../priorities/util/topologies.go:25-70,
# vendor/k8s.io/apimachinery/pkg/apis/meta/v1/helpers.go (LabelSelectorAsSelector), pkg/scheduler/plugins/util/util.go:37-85.
# ----------------------------------------------------------------------------------------------
def _term_props(owner: Pod, term: PodAffinityTerm):
    """(namespaces, selector) of a term: GetNamespacesFromPodAffinityTerm + LabelSelectorAsSelector, canonical + hashable."""
    ns = frozenset(term.namespaces) if term.namespaces else frozenset([owner.namespace])
    if term.nil_selector:
        return (ns, None)
    reqs = [(k, "In", (v,)) for k, v in sorted(term.match_labels.items())]
    for (k, op, vals) in term.match_expressions:
        assert op in ("In", "NotIn", "Exists", "DoesNotExist"), f"label selector operator {op}"
        if op in ("In", "NotIn"):
            assert len(vals) > 0, "In / NotIn need values (LabelSelectorAsSelector returns an error otherwise)"
        else:
            assert len(vals) == 0
        reqs.append((k, op, tuple(sorted(vals))))
    return (ns, tuple(reqs))


def _props_match(pod: Pod, props) -> bool:
    """priorityutil.PodMatchesTermsNamespaceAndSelector (topologies.go:38-49)."""
    ns, reqs = props
    if pod.namespace not in ns:
        return False
    if reqs is None:            # labels.Nothing()
        return False
    return all(_match_requirement(pod.labels, k, op, vals) for (k, op, vals) in reqs)


def _aff_sig(p: Pod):
    def spec(a):
        if a is None:
            return None
        def term(t):
            return (t.topology_key, tuple(sorted(t.match_labels.items())), tuple((k, op, tuple(v)) for (k, op, v) in t.match_expressions),
                    tuple(t.namespaces), t.nil_selector)
        return (tuple(term(t) for t in a.required), tuple((w, term(t)) for (w, t) in a.preferred))
    return (p.namespace, tuple(sorted(p.labels.items())), spec(p.pod_affinity), spec(p.pod_anti_affinity))


def flatten_pod_affinity(nodes, pending, existing, s, on_node, status_of, in_session_job):
    """-> (dict mirroring kb_pod_affinity, dict of the raw objects for object-level checkers).  `pending`: the snapshot's tasks in task
    order; `existing`: pods with a node of the session that are not Pending; on_node: ids of pods node.AddTask accepted."""
    N, T = len(nodes), len(pending)
    nidx = {n.name: i for i, n in enumerate(nodes)}
    listed = [p for p in existing if status_of(p) in ("Bound", "Binding", "Running", "Allocated") and in_session_job(p)]
    for p in listed:
        assert id(p) in on_node, "a listed pod that its node refused (over-committed node): nodeInfo.Filter would hide it from its own node only"
    in_tasks = [p for p in existing if id(p) in on_node]

    # ---- key sets / domains ----
    keysets: Dict[Tuple[str, ...], int] = {}
    dom_rows: List[np.ndarray] = []
    dom_count: List[int] = []

    def keyset_of(keys) -> int:
        ks = tuple(sorted(set(keys)))
        assert all(ks), "an empty topologyKey in a required term is an error in the reference (predicates.go:1311-1313); preferred terms with one never match"
        if ks not in keysets:
            keysets[ks] = len(keysets)
            vals: Dict[Tuple[str, ...], int] = {}
            row = np.full(N, -1, dtype=np.int32)
            for i, n in enumerate(nodes):
                if all(k in n.labels for k in ks):
                    v = tuple(n.labels[k] for k in ks)
                    row[i] = vals.setdefault(v, len(vals))
            dom_rows.append(row)
            dom_count.append(len(vals))
        return keysets[ks]

    # ---- pod types (namespace, labels, affinity spec): all matching is done between types ----
    types: Dict[Tuple, int] = {}
    reps: List[Pod] = []

    def type_of(p: Pod) -> int:
        sg = _aff_sig(p)
        if sg not in types:
            types[sg] = len(types)
            reps.append(p)
        return types[sg]

    ptype = [type_of(p) for p in pending]
    ltype = [type_of(p) for p in listed]
    ttype = [type_of(p) for p in in_tasks]
    NTY = len(reps)

    def req_terms(p, anti):
        a = p.pod_anti_affinity if anti else p.pod_affinity
        return list(a.required) if a is not None else []

    # ---- predicate groups ----
    groups: Dict[Tuple, int] = {}
    g_keyset: List[int] = []
    g_member = []                  # per group: function(type id) -> bool, cached as a list over types
    pend_types = sorted(set(ptype))

    def group_of(key, ks, member_fn):
        if key not in groups:
            groups[key] = len(groups)
            g_keyset.append(ks)
            g_member.append([bool(member_fn(reps[ty])) for ty in range(NTY)])
        return groups[key]

    forbid_ty = {ty: 0 for ty in pend_types}
    need_ty = {ty: -1 for ty in pend_types}
    self_ty = {ty: False for ty in pend_types}
    # (A) required anti-affinity terms pods own: symmetric check (satisfiesExistingPodsAntiAffinity, predicates.go:1400-1439)
    owner_types = sorted(set(ltype) | set(ptype))
    for oty in owner_types:
        owner = reps[oty]
        for term in req_terms(owner, True):
            if not term.topology_key:
                continue            # node.Labels[""] never exists: the term can reject nothing (:1366)
            props = _term_props(owner, term)
            victims = [ty for ty in pend_types if _props_match(reps[ty], props)]
            if not victims:
                continue
            akey = ("A", props, term.topology_key)
            def owns(x, props=props, key=term.topology_key):
                return any(_term_props(x, t) == props and t.topology_key == key for t in req_terms(x, True))
            g = group_of(akey, keyset_of([term.topology_key]), owns)
            for ty in victims:
                forbid_ty[ty] |= 1 << g
    # (B) the pending pods' own required terms (satisfiesPodsAffinityAntiAffinity slow path, :1516-1562)
    for ty in pend_types:
        p = reps[ty]
        for anti in (False, True):
            terms = req_terms(p, anti)
            if not terms:
                continue
            props = frozenset(_term_props(p, t) for t in terms)
            ks = keyset_of([t.topology_key for t in terms])
            g = group_of(("B", props, ks), ks, lambda x, props=props: all(_props_match(x, pr) for pr in props))
            if anti:
                forbid_ty[ty] |= 1 << g
            else:
                need_ty[ty] = g
                self_ty[ty] = all(_props_match(p, pr) for pr in props)      # targetPodMatchesAffinityOfPod(pod, pod)
    NG = len(groups)          # forbid_ty / contrib_ty are bit sets over all NG groups: bits 0..63 go to the masks, the rest to task_xgroup
    g_off = np.zeros(NG + 1, dtype=np.int64)
    for g in range(NG):
        g_off[g + 1] = g_off[g] + dom_count[g_keyset[g]]
    count0 = np.zeros(int(g_off[NG]), dtype=np.int32)
    total0 = np.zeros(NG, dtype=np.int32)
    for p, ty in zip(listed, ltype):
        n = nidx[p.node_name]
        for g in range(NG):
            if g_member[g][ty]:
                total0[g] += 1
                d = dom_rows[g_keyset[g]][n]
                if d >= 0:
                    count0[g_off[g] + d] += 1
    contrib_ty = {ty: sum((1 << g) for g in range(NG) if g_member[g][ty]) for ty in pend_types}

    # ---- priority kinds + weights (interpod_affinity.go:119-171) ----
    def pref_terms(p, anti):
        a = p.pod_anti_affinity if anti else p.pod_affinity
        return list(a.preferred) if a is not None else []

    def weights(P: Pod, X: Pod) -> Dict[str, int]:
        """incoming pod P, existing pod X -> {topologyKey: weight} (processPod)."""
        w: Dict[str, int] = {}
        def add(key, v):
            if key and v:
                w[key] = w.get(key, 0) + v
        for (wt, t) in pref_terms(P, False):
            if _props_match(X, _term_props(P, t)):
                add(t.topology_key, wt)
        for (wt, t) in pref_terms(P, True):
            if _props_match(X, _term_props(P, t)):
                add(t.topology_key, -wt)
        if X.pod_affinity is not None:
            for t in X.pod_affinity.required:                       # hardPodAffinityWeight = 1 (nodeorder.go:159)
                if _props_match(P, _term_props(X, t)):
                    add(t.topology_key, 1)
            for (wt, t) in X.pod_affinity.preferred:
                if _props_match(P, _term_props(X, t)):
                    add(t.topology_key, wt)
        if X.pod_anti_affinity is not None:
            for (wt, t) in X.pod_anti_affinity.preferred:
                if _props_match(P, _term_props(X, t)):
                    add(t.topology_key, -wt)
        return {k: v for k, v in w.items() if v}

    wtab = {(pt, xt): weights(reps[pt], reps[xt]) for pt in pend_types for xt in range(NTY)}
    kinds: Dict[Tuple, int] = {}
    kind_unbound: List[int] = []

    def kind_of(xt: int, unbound: bool) -> int:
        vec = tuple(tuple(sorted(wtab[(pt, xt)].items())) for pt in pend_types)
        if not any(vec):
            return -1
        k = (vec, unbound)
        if k not in kinds:
            kinds[k] = len(kinds)
            kind_unbound.append(1 if unbound else 0)
        return kinds[k]

    xkind = [kind_of(ty, False) for ty in ttype]                    # pods already on nodes: Spec.NodeName is set
    pkind_ty = {ty: kind_of(ty, True) for ty in pend_types}          # a task placed this session: Spec.NodeName stays ""
    NK = len(kinds)
    kc0 = np.zeros((max(1, NK), N), dtype=np.int32)
    for p, k in zip(in_tasks, xkind):
        if k >= 0:
            kc0[k, nidx[p.node_name]] += 1
    kind_rep: Dict[int, int] = {}
    for ty, k in list(zip(ttype, xkind)) + [(ty, pkind_ty[ty]) for ty in pend_types]:
        if k >= 0:
            kind_rep.setdefault(k, ty)
    wlist_ty = {}
    for pt in pend_types:
        lst = []
        for k in range(NK):
            for key, v in sorted(wtab[(pt, kind_rep[k])].items()):
                lst.append((k, keyset_of([key]), v))
        wlist_ty[pt] = lst
    w_off = np.zeros(T + 1, dtype=np.uint32)
    wk, wks, wv = [], [], []
    for t in range(T):
        for (k, ks, v) in wlist_ty[ptype[t]]:
            wk.append(k); wks.append(ks); wv.append(v)
        w_off[t + 1] = len(wk)

    for t in range(T):
        ty = ptype[t]
        p = pending[t]
        if p.pod_affinity is not None or p.pod_anti_affinity is not None:
            s.task_flags[t] |= abi.KB_TASK_HAS_POD_AFFINITY
        if self_ty[ty]:
            s.task_flags[t] |= abi.KB_TASK_AFF_SELF_MATCH
    if any(p.pod_affinity is not None or p.pod_anti_affinity is not None for p in existing):
        s.flags = int(getattr(s, "flags", 0)) | abi.KB_SNAPSHOT_PLACED_POD_AFFINITY

    M64 = (1 << 64) - 1

    def xgroups(ty):
        f, c = forbid_ty[ty] >> 64, contrib_ty[ty] >> 64
        return [((64 + i) << 2) | ((f >> i) & 1) * abi.KB_XGROUP_FORBID | ((c >> i) & 1) * abi.KB_XGROUP_CONTRIB
                for i in range(max(f.bit_length(), c.bit_length())) if ((f | c) >> i) & 1]

    NKS = len(keysets)
    pa = {
        "n_keysets": NKS, "n_groups": NG, "n_kinds": NK, "n_weights": len(wk), "first_unbound_node": -1,
        "node_domain": np.stack(dom_rows).astype(np.int32) if NKS else np.zeros((1, max(1, N)), dtype=np.int32),
        "keyset_domains": np.array(dom_count if NKS else [0], dtype=np.uint32),
        "group_keyset": np.array(g_keyset if NG else [0], dtype=np.uint32),
        "group_count0": count0 if count0.size else np.zeros(1, dtype=np.int32),
        "group_total0": total0 if NG else np.zeros(1, dtype=np.int32),
        "task_forbid": np.array([forbid_ty[ty] & M64 for ty in ptype] or [0], dtype=np.uint64),
        "task_need": np.array([need_ty[ty] for ty in ptype] or [-1], dtype=np.int32),
        "task_contrib": np.array([contrib_ty[ty] & M64 for ty in ptype] or [0], dtype=np.uint64),
        "task_kind": np.array([pkind_ty[ty] for ty in ptype] or [-1], dtype=np.int32),
        "node_kind_count0": kc0,
        "kind_unbound": np.array(kind_unbound or [0], dtype=np.uint8),
        "task_weight_off": w_off,
        "weight_kind": np.array(wk or [0], dtype=np.int32),
        "weight_keyset": np.array(wks or [0], dtype=np.int32),
        "weight_value": np.array(wv or [0], dtype=np.int64),
    }
    if NG > 64:               # groups >= 64: per task the entries (g << 2) | KB_XGROUP_FORBID | KB_XGROUP_CONTRIB
        xl = [xgroups(ty) for ty in ptype]
        pa["task_xgroup_off"] = np.concatenate([[0], np.cumsum([len(x) for x in xl], dtype=np.int64)]).astype(np.uint32)
        pa["task_xgroup"] = np.array([e for x in xl for e in x] or [0], dtype=np.uint32)

    # ---- the raw objects (what a checker that walks the pods one by one needs): pending pods in task order, then the others ----
    lset, tset = set(id(p) for p in listed), set(id(p) for p in in_tasks)
    pa["member_pod_ids"] = set(id(p) for p, ty in zip(listed, ltype) if any(g_member[g][ty] for g in range(NG)))   # -> KB_RUNNING_AFF_MEMBER
    pa["member_groups"] = {id(p): [g for g in range(NG) if g_member[g][ty]] for p, ty in zip(listed, ltype)}     # -> kb_running.aff_group
    ob = {"nodes": nodes, "pending": list(pending), "existing": list(existing), "node_index": nidx,
          "listed": [id(p) in lset for p in existing], "in_tasks": [id(p) in tset for p in existing]}
    return pa, ob
