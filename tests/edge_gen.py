"""Seeded sessions whose node states sit on the boundaries of the fit and score arithmetic, built from objects
(builder.SessionBuilder -> flatten(W=2): cpu, memory and nvidia.com/gpu, so R = 3 / W = 2 and the sessions run on cycle_kernel).

synth.generate clusters never get there: three node shapes, power-of-two requests, no node at its pod cap, no Idle below 0, at
most ~20 placements of one job on one node.  Each part of edge_session() sets up one kind of edge on purpose, most of them on
nodes that a nodeSelector reserves for one PodGroup, so that the run of that group walks the node's state down a known path:
  epsilon fits     Idle = k * request + delta: the k-th placement fits exactly, through the 10 m / 10 Mi epsilon, or not at all;
                   and nodes whose Running pods already fit only through the epsilon (Idle in [-9, 0) m at load)
  pod caps         max_pods - pods in {0, 1, 3, 4, 5, 7, 8, 9, 35, 36, 37, 39, 40, 41}: around the placement depths the replay
                   evaluates up front for patched (4) and list (8) candidates and the end of the first chain extension (8 + 32)
  flips            terminating pods: a run Allocates k times, Pipelines m times onto Releasing, then stops fitting
  capacities       system-reserved allocatable (7910m / 32879468Ki), memory up to 24 Ti, zero cpu or zero memory, pods without a
                   cpu / memory request (the non-zero defaults), non-zero sums beyond allocatable
  scalars          nvidia.com/gpu requests of exactly 10 milli (skipped by LessEqual) and 11 milli, on nodes with and without GPUs
  long runs        PodGroups of 50..150 identical tasks: on one node (> 40 placements in a run: a second chain extension), and
                   alternating over 2..4 identical nodes (several candidates past depth 8 at once, their extensions evict each other)
  pool builder     a mix of minMember values (jobs yield and come back: the pool built ahead misses) and runs of one class
coverage() measures what the ORACLE did with a session, so that a test can assert that the edges were really reached."""
from __future__ import annotations

import numpy as np

from kube_batch_b200 import abi
from kube_batch_b200 import builder as B
from kube_batch_b200.snapshot import PluginConf

MI, GI, TI = 1 << 20, 1 << 30, 1 << 40
GPU = B.GPU
FPGA = "example.com/fpga"
MIN_MEM = 10 * MI
CAP_SLACK = [0, 1, 3, 4, 5, 7, 8, 9, 35, 36, 37, 39, 40, 41]


class _Gen:
    def __init__(self, seed, queues, wide, pref):
        self.rng = np.random.default_rng(seed)
        self.b = B.SessionBuilder()
        self.queues = [f"q{i}" for i in range(queues)]
        for i, q in enumerate(self.queues):
            self.b.add_queue(B.Queue(q, int(self.rng.integers(1, 4)), creation=i))
        self.wide, self.pref = wide, pref
        self.nodes = []          # [name, alloc dict, labels, running pods, pod slack]
        self.n_groups = 0
        self.n_running = 0
        self.run_groups = []
        for i in range(3):       # the Running pods' PodGroups (their own queues, priorities)
            g = self.group(min_member=0, priority=int(self.rng.integers(0, 3)), name=f"run{i}")
            self.run_groups.append(g)

    # ---- objects ----
    def node(self, cpu_m, mem, gpu=0, labels=None, slack=110):
        name = f"n{len(self.nodes):04d}"
        alloc = {"cpu": cpu_m / 1000.0, "memory": float(mem)}
        if gpu:
            alloc[GPU] = gpu
        if self.wide and self.rng.random() < 0.5:
            alloc[FPGA] = 2
        lab = {"zone": "abc"[len(self.nodes) % 3]}
        lab.update(labels or {})
        self.nodes.append([name, alloc, lab, [], slack])
        return self.nodes[-1]

    def group(self, min_member, priority=0, name=None):
        name = name or f"g{self.n_groups:03d}"
        self.n_groups += 1
        self.b.add_pod_group(B.PodGroup("ns", name, str(self.rng.choice(self.queues)), min_member=min_member, priority=priority,
                                        creation=int(self.rng.integers(0, 4))))
        return name

    def running(self, node, req, deleting=False):
        g = str(self.rng.choice(self.run_groups))
        node[3].append(B.Pod("ns", f"run-{self.n_running:05d}", node[0], "Running", dict(req), group=g,
                             priority=int(self.rng.integers(0, 3)), creation=self.n_running, deleting=deleting))
        self.n_running += 1

    def tasks(self, group, count, req, selector=None, prefix=None, preferred=None, priority=None):
        for k in range(count):
            self.b.add_pod(B.Pod("ns", f"{prefix or group}-p{k:03d}", "", "Pending", dict(req), group=group, creation=k,
                                 node_selector=dict(selector or {}), preferred_terms=list(preferred or []), priority=priority))

    def finish(self, W):
        for name, alloc, labels, pods, slack in self.nodes:
            alloc = dict(alloc)
            alloc["pods"] = len(pods) + slack
            self.b.add_node(B.Node(name, alloc, labels=labels))
            for p in pods:
                self.b.add_pod(p)
        return self.b.flatten(W=W)


def _req(cpu_m=None, mem=None, gpu_m=None):
    r = {}
    if cpu_m is not None:
        r["cpu"] = cpu_m / 1000.0
    if mem is not None:
        r["memory"] = float(mem)
    if gpu_m is not None:
        r[GPU] = gpu_m / 1000.0
    return r


def edge_session(seed: int, n_plain: int = 24, queues: int = 1, wide: bool = False, pref: bool = False, long_runs: bool = True,
                 best_effort: bool = False):
    """One boundary-state session.  wide: a fourth resource and W = 3 (R = 4: the per-visit kernels).  pref: preferred
    node-affinity terms on some groups (cycle_kernel<3,2,1>).  best_effort: pods with an empty request as well (backfill)."""
    G = _Gen(seed, queues, wide, pref)
    rng = G.rng
    pref_terms = [(int(rng.choice([1, 20, 50])), [("zone", "In", [str(rng.choice(list("abc")))])])] if pref else None

    # ---- the general population: plain, system-reserved, huge, zero-capacity nodes with random fillers and pod slack ----
    shapes = [(32000, 128 * GI, 4), (7910, 32879468 * 1024, 0), (96000, int(rng.choice([4, 24])) * TI, 8), (0, 64 * GI, 0),
              (16000, 0, 0), (32000, 128 * GI, 0)]
    for i in range(n_plain):
        cpu, mem, gpu = shapes[i % len(shapes)] if i < 2 * len(shapes) else shapes[int(rng.choice([0, 0, 1, 2, 5]))]
        zero = {"zero": "cpu"} if cpu == 0 else ({"zero": "mem"} if mem == 0 else {})
        nd = G.node(cpu, mem, gpu, slack=int(rng.choice(CAP_SLACK + [110, 110])), labels=zero)
        for _ in range(int(rng.integers(0, 4))):
            G.running(nd, _req(int(rng.integers(1, 900)), int(rng.integers(1, 3 * GI))))
        if i % 5 == 4 and cpu and mem:        # Running pods that fit only through the epsilon: Idle starts in [-9, 0) m / (-10 Mi, 0)
            used_c = sum(B.SessionBuilder._milli(p.requests.get("cpu", 0)) for p in nd[3])
            used_m = sum(p.requests.get("memory", 0) for p in nd[3])
            if i % 10 == 4:
                G.running(nd, _req(cpu - used_c + int(rng.integers(1, 10)), int(rng.integers(1, GI))))
            else:
                G.running(nd, _req(int(rng.integers(1, 100)), mem - used_m + int(rng.integers(1, MIN_MEM))))

    # ---- epsilon fits: Idle = k * req + delta on a node reserved for one group of k + 2 identical tasks ----
    for e in range(6):
        k = int(rng.choice([1, 2, 3, 4, 5, 8, 9, 12, 40, 41]))
        rc = int(rng.choice([100, 250, 333, 1000, 7]))
        rm = int(rng.choice([128 * MI, 200 * MI, 333 * MI + 17, GI]))
        on_cpu = e % 2 == 0
        delta = [0, -9, -10][e // 2] if on_cpu else [0, -MIN_MEM + 1, -MIN_MEM][e // 2]
        cpu_alloc, mem_alloc = 64000 + int(rng.integers(0, 999)), 512 * GI + int(rng.integers(0, 12345))
        nd = G.node(cpu_alloc, mem_alloc, slack=110, labels={"eps": str(e)})
        want_c = k * rc + delta if on_cpu else k * rc + 5000
        want_m = k * rm + 3 * GI if on_cpu else k * rm + delta
        G.running(nd, _req(cpu_alloc - want_c, mem_alloc - want_m))
        g = G.group(min_member=k + 2)
        G.tasks(g, k + 2, _req(rc, rm), selector={"eps": str(e)})

    # ---- pod caps on reserved nodes: the run stops at max_pods partway ----
    for c, slack in enumerate(rng.choice(CAP_SLACK, 5, replace=False).tolist()):
        nd = G.node(64000, 256 * GI, slack=int(slack), labels={"cap": str(c)})
        for _ in range(int(rng.integers(0, 3))):
            G.running(nd, _req(int(rng.integers(1, 500)), int(rng.integers(1, GI))))
        g = G.group(min_member=int(slack) + 3)
        G.tasks(g, int(slack) + 3, _req(50, 64 * MI), selector={"cap": str(c)})

    # ---- Allocate -> Pipeline flips: Idle = k * req, Releasing = m * req, k + m + 2 tasks ----
    for f in range(3):
        k, m = int(rng.choice([1, 3, 4, 7, 8, 9, 12, 39])), int(rng.integers(1, 7))
        rc, rm = int(rng.choice([200, 500, 1000])), int(rng.choice([256 * MI, GI]))
        cpu_alloc, mem_alloc = 96000, 384 * GI
        nd = G.node(cpu_alloc, mem_alloc, slack=110, labels={"flip": str(f)})
        G.running(nd, _req(m * rc, m * rm), deleting=True)
        G.running(nd, _req(cpu_alloc - m * rc - k * rc, mem_alloc - m * rm - k * rm - int(rng.integers(0, MI))))
        g = G.group(min_member=k + m + 2)
        G.tasks(g, k + m + 2, _req(rc, rm), selector={"flip": str(f)})

    # ---- scalar requests of 10 m (skipped) and 11 m, no cpu / no memory request (the non-zero defaults), zero-capacity nodes ----
    for gpu_m in (10, 11):
        g = G.group(min_member=int(rng.choice([0, 1, 3])))
        G.tasks(g, int(rng.integers(3, 9)), _req(int(rng.choice([10, 100])), 64 * MI, gpu_m))
    g = G.group(min_member=1)
    G.tasks(g, 6, _req(mem=128 * MI), prefix=g + "-nocpu")
    G.tasks(g, 6, _req(cpu_m=5), prefix=g + "-nomem")
    for axis, req in (("cpu", _req(mem=128 * MI)), ("mem", _req(cpu_m=250))):       # only a zero-capacity node is feasible
        g = G.group(min_member=int(rng.choice([1, 4])))
        G.tasks(g, 4, req, selector={"zero": axis})
    if best_effort:
        g = G.group(min_member=int(rng.choice([0, 2])))
        G.tasks(g, 8, {}, prefix=g + "-be")

    # ---- long runs ----
    if long_runs:
        nd = G.node(128000, 1 * TI, slack=int(rng.choice([150, 60])), labels={"solo": "0"})     # one feasible node
        g = G.group(min_member=150)
        G.tasks(g, int(rng.integers(50, 151)), _req(100, 128 * MI), selector={"solo": "0"})
        for t in range(2):                                                                       # 2..4 identical nodes
            width = int(rng.integers(2, 5))
            for _ in range(width):
                G.node(64000, 256 * GI, slack=110, labels={"twin": str(t)})
            g = G.group(min_member=150)
            G.tasks(g, int(rng.integers(10, 38)) * width, _req(100, 128 * MI), selector={"twin": str(t)})
        for r in range(2):        # relays: jobs of one class in a row on one node (the next job's list is patched, then run deep)
            G.node(64000, 256 * GI, slack=110, labels={"relay": str(r)})
            for _ in range(int(rng.integers(2, 4))):
                g = G.group(min_member=150)
                G.tasks(g, int(rng.integers(3, 25)), _req(200, 256 * MI), selector={"relay": str(r)})
        for _ in range(2):                                                                        # unconstrained long runs
            g = G.group(min_member=int(rng.choice([50, 150])))
            G.tasks(g, int(rng.integers(50, 151)), _req(int(rng.choice([100, 250])), int(rng.choice([128, 256])) * MI))

    # ---- the pool builder: many small jobs of mixed minMember (some yield after one task and come back) ----
    for _ in range(int(rng.integers(8, 16))):
        size = int(rng.integers(1, 12))
        g = G.group(min_member=int(rng.choice([0, 1, size // 2, size])), priority=int(rng.integers(0, 3)))
        rc = int(rng.choice([100, 250, 500, 1000, 1500, 4000]))
        G.tasks(g, size, _req(rc, int(rng.choice([128 * MI, 512 * MI, 2 * GI, 333 * MI + 5]))),
                preferred=pref_terms if (pref and rng.random() < 0.5) else None, priority=int(rng.integers(0, 3)))
    snap = G.finish(W=3 if wide else 2)
    assert (snap.R, snap.W) == ((4, 3) if wide else (3, 2)), (snap.R, snap.W)
    return snap


def mostrequested_conf():
    """Binpacking: a run stays on one node until it is full (the long chains of a single candidate)."""
    return PluginConf.from_names([["priority", "gang"], ["drf", "predicates", "proportion", "nodeorder"]],
                                 {"nodeorder": {"leastrequested.weight": "0", "mostrequested.weight": "1", "balancedresource.weight": "0"}})


def coverage(snap, o) -> dict:
    """What the oracle's decisions and final state reached.  A run = consecutive placement steps of one job."""
    d = o.decisions
    job = snap.job_of_task()
    placed = np.nonzero(d["node"] >= 0)[0]
    placed = placed[np.argsort(d["step"][placed], kind="stable")]
    max_on_one = 0
    multi_deep = 0
    flips = 0
    i = 0
    while i < len(placed):
        j = i
        while j < len(placed) and job[placed[j]] == job[placed[i]]:
            j += 1
        run = placed[i:j]
        nodes, counts = np.unique(d["node"][run], return_counts=True)
        max_on_one = max(max_on_one, int(counts.max()))
        if int((counts > 8).sum()) >= 2:
            multi_deep += 1
        alloc_nodes = set(d["node"][run][d["kind"][run] == abi.KB_KIND_ALLOCATED].tolist())
        flips += int(sum(1 for t in run if d["kind"][t] == abi.KB_KIND_PIPELINED and int(d["node"][t]) in alloc_nodes))
        i = j
    touched = np.zeros(snap.N, dtype=bool)
    touched[d["node"][placed]] = True
    idle = o.node_idle
    zero_cap = (snap.node_alloc_cpu == 0) | (snap.node_alloc_mem == 0)
    return dict(
        max_run_on_one_node=max_on_one,
        runs_with_two_deep_nodes=multi_deep,
        nodes_at_pod_cap=int(((o.node_pods == snap.node_max_pods) & touched).sum()),
        nodes_idle_cpu_in_epsilon=int(((idle[0] >= -9) & (idle[0] < 0)).sum()),
        nodes_idle_mem_in_epsilon=int(((idle[1] > -MIN_MEM) & (idle[1] < 0)).sum()),
        pipelined_after_allocate_in_run=flips,
        nodes_nz_over_allocatable=int(((o.node_nz_cpu > snap.node_alloc_cpu) | (o.node_nz_mem > snap.node_alloc_mem)).sum()),
        zero_capacity_nodes_used=int((zero_cap & touched).sum()),
    )


def assert_covered(cov: dict, what: str, long_runs: bool = True):
    """Every edge of the module docstring reached at least once."""
    need = dict(cov)
    if not long_runs:
        need.pop("max_run_on_one_node")
        need.pop("runs_with_two_deep_nodes")
    else:
        assert cov["max_run_on_one_node"] > 40, (what, cov)
    assert all(v > 0 for v in need.values()), (what, cov)


def merge(covs):
    out = {}
    for c in covs:
        for k, v in c.items():
            out[k] = max(out.get(k, 0), v) if k == "max_run_on_one_node" else out.get(k, 0) + v
    return out
