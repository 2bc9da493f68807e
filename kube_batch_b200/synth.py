"""Seeded synthetic Session snapshots for the BASELINE.json configurations (SURVEY.md §8d).

There is no network and no cluster: these snapshots stand in for cache.Snapshot()
(kube-batch/pkg/scheduler/cache/cache.go:627-683) of a kubemark-like cluster.  The generator is
deterministic in (config, seed); seed = 0xB200 + config number by default (PCG64).

Label / taint / port atoms (the interning a flattener would do; include/kbgpu.h):
  label word0 bit0..2 : zone in {a,b,c};   label word1 bit5 : disk=ssd
  taint word0 bit0    : dedicated=batch:NoSchedule
  port  word0 bit0    : (0.0.0.0, TCP, 8080)
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import numpy as np

from . import abi
from .snapshot import PluginConf, PluginOption, Snapshot

GiB = 1 << 30
NODE_SHAPES = [(32000, 128 * GiB, 0), (64000, 256 * GiB, 8000), (96000, 384 * GiB, 8000)]
NODE_PROBS = [0.5, 0.3, 0.2]
TASK_CPU = [500, 1000, 2000, 4000]
TASK_MEM = [1 * GiB, 2 * GiB, 4 * GiB, 8 * GiB]


@dataclass
class SynthSpec:
    name: str
    tasks: int
    jobs: int
    nodes: int
    queues: int = 1
    min_member_frac: float = 1.0     # minMember = ceil(frac * tasks_in_job)
    homogeneous_nodes: bool = False  # C5: one node shape
    oversub: float = 1.3             # demand / free capacity on the scarcest of cpu, mem
    hetero_job_frac: float = 0.0     # fraction of jobs whose tasks are NOT identical
    prio_levels: int = 1
    R: int = 3                       # resource dims: cpu, memory, nvidia.com/gpu, then extra scalars
    W: int = 2                       # 64-bit words per label / taint / port mask
    seed: Optional[int] = None
    conf: Optional[PluginConf] = None


def conf_c1() -> PluginConf:
    # "allocate+gang+predicates" (+priority), explicit flags like the reference tests pass them
    return PluginConf([[PluginOption("priority", enabled_job_order=True, enabled_task_order=True),
                        PluginOption("gang", enabled_job_order=True, enabled_job_ready=True, enabled_job_pipelined=True)],
                       [PluginOption("predicates", enabled_predicate=True)]])


def conf_c2() -> PluginConf:
    return PluginConf.from_names([["gang"], ["drf", "predicates", "nodeorder"]])


def conf_default() -> PluginConf:
    return PluginConf.default()


CONFIGS: Dict[str, SynthSpec] = {
    "c1": SynthSpec("c1", tasks=9, jobs=3, nodes=10, seed=0xB200 + 1),
    "c2": SynthSpec("c2", tasks=1000, jobs=100, nodes=500, seed=0xB200 + 2),
    "c3": SynthSpec("c3", tasks=50_000, jobs=5_000, nodes=5_000, seed=0xB200 + 3),
    "c4": SynthSpec("c4", tasks=200_000, jobs=20_000, nodes=20_000, queues=8, seed=0xB200 + 4),
    "c5": SynthSpec("c5", tasks=1_000_000, jobs=100_000, nodes=100_000, homogeneous_nodes=True, seed=0xB200 + 5),
}


def config_conf(name: str) -> PluginConf:
    if name == "c1":
        return conf_c1()
    if name == "c2":
        return conf_c2()
    if name == "c5":
        return PluginConf.from_names([["gang"], ["drf", "predicates", "nodeorder"]])
    return conf_default()


def generate(spec: SynthSpec) -> Snapshot:
    rng = np.random.Generator(np.random.PCG64(spec.seed if spec.seed is not None else 0xB200))
    R, W = spec.R, spec.W
    assert 3 <= R <= abi.KB_MAX_R and 2 <= W <= abi.KB_MAX_W
    N, Jp, Q = spec.nodes, spec.jobs, spec.queues
    # pending tasks per job
    base = spec.tasks // Jp
    per_job = np.full(Jp, base, dtype=np.int64)
    per_job[: spec.tasks - base * Jp] += 1
    T = int(per_job.sum())
    n_fill = max(1, N // 16)          # filler jobs owning the pre-existing Running tasks
    J = Jp + n_fill
    s = Snapshot(R, W, N, T, J, Q)

    # ---------------- nodes ----------------
    if spec.homogeneous_nodes:
        shape_id = np.ones(N, dtype=np.int64)
    else:
        shape_id = rng.choice(3, size=N, p=NODE_PROBS)
    shapes = np.array(NODE_SHAPES, dtype=np.float64)
    alloc = np.zeros((R, N))
    alloc[:3] = shapes[shape_id].T                        # [R][N]
    present = np.where(alloc[2] > 0, 1 << 2, 0).astype(np.uint32)
    for r in range(3, R):                                 # extra scalar resources on a third of the nodes
        has = rng.random(N) < 0.33
        alloc[r] = np.where(has, 4000.0, 0.0)
        present |= np.where(has, 1 << r, 0).astype(np.uint32)
    s.node_allocatable[:] = alloc
    s.node_alloc_present[:] = present
    s.node_alloc_cpu[:] = alloc[0].astype(np.int64)
    s.node_alloc_mem[:] = alloc[1].astype(np.int64)
    s.node_max_pods[:] = 110
    zone = rng.integers(0, 3, size=N)
    s.node_labels[0] = (np.uint64(1) << zone.astype(np.uint64))
    s.node_labels[W - 1] = np.where(rng.random(N) < 0.5, np.uint64(1) << np.uint64(5), np.uint64(0))
    s.node_taints[0] = np.where(rng.random(N) < 0.05, np.uint64(1), np.uint64(0))
    if W > 2:                                             # a second taint atom in the last word
        s.node_taints[W - 1] = np.where(rng.random(N) < 0.03, np.uint64(1) << np.uint64(9), np.uint64(0))
    s.node_ports[0] = np.where(rng.random(N) < 0.01, np.uint64(1), np.uint64(0))
    flags = np.zeros(N, dtype=np.uint32)
    u = rng.random(N)
    flags[u < 0.004] |= abi.KB_NODE_UNSCHEDULABLE
    flags[(u >= 0.004) & (u < 0.006)] |= abi.KB_NODE_NET_UNAVAILABLE
    flags[(u >= 0.006) & (u < 0.01)] |= abi.KB_NODE_MEM_PRESSURE
    s.node_flags[:] = flags

    # ---------------- pending jobs / tasks ----------------
    job_cpu = rng.choice(TASK_CPU, size=Jp)
    job_mem = rng.choice(TASK_MEM, size=Jp)
    job_gpu = np.where(rng.random(Jp) < 0.2, 1000, 0)
    uj = rng.random(Jp)
    job_zone = np.where(uj < 0.10, rng.integers(0, 3, size=Jp), -1)
    job_aff = (uj >= 0.10) & (uj < 0.13)        # required node affinity: (zone a AND ssd) OR (zone b)
    job_tol = rng.random(Jp) < 0.05
    job_port = rng.random(Jp) < 0.02
    hetero = rng.random(Jp) < spec.hetero_job_frac

    off = np.zeros(J + 1, dtype=np.int64)
    off[1:Jp + 1] = np.cumsum(per_job)
    off[Jp + 1:] = T
    s.job_task_off[:] = off.astype(np.uint32)
    tj = np.repeat(np.arange(Jp), per_job)               # job of each task
    cpu = job_cpu[tj].astype(np.float64)
    mem = job_mem[tj].astype(np.float64)
    gpu = job_gpu[tj].astype(np.float64)
    if hetero.any():
        ht = hetero[tj]
        cpu = np.where(ht, rng.choice(TASK_CPU, size=T), cpu)
        mem = np.where(ht, rng.choice(TASK_MEM, size=T), mem)
    s.task_resreq[0], s.task_resreq[1], s.task_resreq[2] = cpu, mem, gpu
    extra_present = np.zeros(T, dtype=np.uint32)
    for r in range(3, R):                                 # ~6 % of the jobs ask for one unit of an extra scalar
        wants = (rng.random(Jp) < 0.06)[tj]
        s.task_resreq[r] = np.where(wants, 1000.0, 0.0)
        extra_present |= np.where(wants, 1 << r, 0).astype(np.uint32)
    s.task_initreq[:] = s.task_resreq
    # a few pods carry an init container larger than the sum of containers (api/pod_info.go:53-73)
    big_init = rng.random(T) < 0.01
    s.task_initreq[0] = np.where(big_init, s.task_initreq[0] + 500, s.task_initreq[0])
    s.task_res_present[:] = (1 << 2) | extra_present      # BuildResourceList always lists nvidia.com/gpu
    s.task_nz_cpu[:] = cpu.astype(np.int64)
    s.task_nz_mem[:] = mem.astype(np.int64)
    zt = job_zone[tj]
    s.task_sel_req[0] = np.where(zt >= 0, np.uint64(1) << np.maximum(zt, 0).astype(np.uint64), np.uint64(0))
    at = job_aff[tj]
    s.task_n_aff_terms[:] = np.where(at, 2, 0)
    s.task_aff_terms[0, 0] = np.where(at, np.uint64(1), np.uint64(0))             # term 0: zone a ...
    s.task_aff_terms[0, W - 1] = np.where(at, np.uint64(1) << np.uint64(5), np.uint64(0))  # ... AND disk=ssd
    s.task_aff_terms[1, 0] = np.where(at, np.uint64(2), np.uint64(0))             # term 1: zone b
    s.task_tol[0] = np.where(job_tol[tj], np.uint64(1), np.uint64(0))
    if W > 2:
        s.task_tol[W - 1] = np.where((rng.random(Jp) < 0.5)[tj], np.uint64(1) << np.uint64(9), np.uint64(0))
    pt = job_port[tj]
    s.task_port_own[0] = np.where(pt, np.uint64(1), np.uint64(0))
    s.task_port_conflict[0] = s.task_port_own[0]
    s.task_prio[:] = 1
    if spec.prio_levels > 1:
        s.task_prio[:] = rng.integers(1, spec.prio_levels + 1, size=T)
    s.task_ctime[:] = tj                                  # pods of a PodGroup share a timestamp -> UID decides
    s.task_uid_rank[:] = rng.permutation(T).astype(np.uint32)

    s.job_min_avail[:Jp] = np.ceil(per_job * spec.min_member_frac).astype(np.int32)
    s.job_queue[:Jp] = rng.integers(0, Q, size=Jp)
    s.job_prio[:] = 0
    if spec.prio_levels > 1:
        s.job_prio[:Jp] = rng.integers(0, spec.prio_levels, size=Jp)
    s.job_ctime[:] = np.arange(J)
    s.job_alloc0_present[:] = 1 << 2
    s.queue_weight[:] = np.arange(1, Q + 1)
    s.queue_ctime[:] = 0

    # ---------------- pre-existing utilisation (Running tasks of filler jobs) ----------------
    cap = alloc.sum(axis=1)
    dem = s.task_resreq.sum(axis=1)
    need = np.array([dem[r] / (spec.oversub * cap[r]) if cap[r] > 0 else 0.0 for r in range(2)])
    util = float(np.clip(1.0 - need.max(), 0.0, 0.98))
    node_util = np.clip(util + rng.uniform(-0.15, 0.15, size=N), 0.0, 0.985)
    # filler pods are 1/64-of-the-node bricks (nz == request: requests are always set)
    brick = np.stack([alloc[0] / 64.0, alloc[1] / 64.0, np.zeros(N)])     # [R][N], integral for every shape
    k = np.floor(node_util * 64.0).astype(np.int64)
    used = np.zeros((R, N))
    used[:3] = brick * k[None, :]
    gpu_used = np.where(alloc[2] > 0, 1000.0 * rng.integers(0, 5, size=N), 0.0)
    used[2] = gpu_used
    s.node_used[:] = used
    s.node_idle[:] = alloc - used
    s.node_pods[:] = k.astype(np.int32)
    s.node_nz_cpu[:] = used[0].astype(np.int64)
    s.node_nz_mem[:] = used[1].astype(np.int64)
    # ~2% of nodes carry one Releasing pod (deleted, still terminating): Idle shrinks, Releasing grows
    rel = (rng.random(N) < 0.02) & (s.node_idle[0] >= 4000) & (s.node_idle[1] >= 8 * GiB)
    relreq = np.zeros(R)
    relreq[0], relreq[1] = 4000.0, 8.0 * GiB
    s.node_releasing[:] = np.where(rel[None, :], relreq[:, None], 0.0)
    s.node_idle[:] -= s.node_releasing
    s.node_used[:] += s.node_releasing
    s.node_pods[:] += rel.astype(np.int32)
    s.node_nz_cpu[:] += (rel * relreq[0]).astype(np.int64)
    s.node_nz_mem[:] += (rel * relreq[1]).astype(np.int64)

    # filler jobs own the Running bricks round-robin
    fj = np.arange(N) % n_fill
    for r in range(R):
        s.job_alloc0[r, Jp:] = np.bincount(fj, weights=used[r], minlength=n_fill)
    ready0 = np.bincount(fj, weights=k, minlength=n_fill).astype(np.int32)
    s.job_ready0[Jp:] = ready0
    s.job_min_avail[Jp:] = ready0
    s.job_queue[Jp:] = np.arange(n_fill) % Q
    s.meta = {"spec": spec.name, "seed": spec.seed, "util": util, "pending_jobs": Jp, "filler_jobs": n_fill}
    s.validate()
    return s


def running_of(s: Snapshot, preemptable_frac: float = 0.0, seed: int = 1) -> dict:
    """The Running tasks behind the filler jobs' aggregates, one by one (kb_running): node n carries node_pods[n] bricks of
    1/64 of the node each (minus its terminating pod, which is Releasing, not Running).  preemptable_frac > 0 lowers MinAvailable
    of that share of the filler jobs IN PLACE so that gang lets reclaim / preempt take some of their pods (gang.go:70-90)."""
    Jp, n_fill = s.meta["pending_jobs"], s.meta["filler_jobs"]
    N, R = s.N, s.R
    rel = (s.node_releasing[0] > 0).astype(np.int64)
    k = s.node_pods.astype(np.int64) - rel
    node = np.repeat(np.arange(N, dtype=np.uint32), k)
    n = int(k.sum())
    resreq = np.zeros((R, n))
    resreq[0] = np.repeat(s.node_allocatable[0] / 64.0, k)
    resreq[1] = np.repeat(s.node_allocatable[1] / 64.0, k)
    rng = np.random.Generator(np.random.PCG64(seed))
    if preemptable_frac > 0:
        loose = rng.random(n_fill) < preemptable_frac
        s.job_min_avail[Jp:] = np.where(loose, np.maximum(1, s.job_ready0[Jp:] // 2), s.job_min_avail[Jp:])
    return {"node": node, "job": (Jp + node % n_fill).astype(np.uint32), "resreq": resreq,
            "res_present": np.full(n, 1 << 2, dtype=np.uint32), "prio": np.ones(n, dtype=np.int32),
            "ctime": np.zeros(n, dtype=np.int64), "uid_rank": rng.permutation(n).astype(np.uint32),
            "flags": np.zeros(n, dtype=np.uint32)}


def make(name: str, replica: int = 0) -> Tuple[Snapshot, PluginConf]:
    """replica > 0: another cluster of the same shape (seed + 1000 * replica) — what rank `replica` schedules when bench.py runs
    N independent sessions on N GPUs."""
    spec = CONFIGS[name]
    if replica:
        from dataclasses import replace
        spec = replace(spec, seed=(spec.seed if spec.seed is not None else 0xB200) + 1000 * int(replica))
    return generate(spec), (spec.conf or config_conf(name))


def add_host_spread(s: Snapshot, frac: float = 0.1, labels: int = 8, seed: int = 7) -> Snapshot:
    """Gives `frac` of the PodGroups the most common inter-pod constraint — "one replica per host": every pod of the group carries the
    label app=<L> (L = one of `labels` values) and a required anti-affinity term {app=<L>, topologyKey kubernetes.io/hostname}.  Fills
    kb_pod_affinity (include/kbgpu.h) exactly as builder.flatten_pod_affinity would for such pods: per label one counter group for
    the term the pods OWN (satisfiesExistingPodsAntiAffinity) and one for the pods that MATCH the term list (the pod's own check) —
    same members, both forbidden to and joined by the label's pods; one key set (hostname: a domain per node); no pod kinds (required
    anti-affinity terms carry no priority weight).  Pods already running carry no labels here.  Label L owns groups 2L and 2L + 1:
    labels 0..31 are bits of the masks, labels >= 32 entries of task_xgroup (only emitted when there are more than 64 groups)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    T, N, J = s.T, s.N, s.J
    forbid = np.zeros(max(T, 1), dtype=np.uint64)
    lab_of = np.full(max(T, 1), -1, dtype=np.int64)
    for j in range(J):
        lo, hi = int(s.job_task_off[j]), int(s.job_task_off[j + 1])
        if hi > lo and rng.random() < frac:
            lab = int(rng.integers(0, labels))
            if lab < 32:
                forbid[lo:hi] = np.uint64(3 << (2 * lab))
            lab_of[lo:hi] = lab
            s.task_flags[lo:hi] |= abi.KB_TASK_HAS_POD_AFFINITY
    G = 2 * labels
    s.pod_affinity = {
        "n_keysets": 1, "n_groups": G, "n_kinds": 0, "n_weights": 0, "first_unbound_node": -1,
        "node_domain": np.arange(max(N, 1), dtype=np.int32).reshape(1, -1), "keyset_domains": np.array([N], dtype=np.uint32),
        "group_keyset": np.zeros(G, dtype=np.uint32), "group_count0": np.zeros(max(1, G * N), dtype=np.int32),
        "group_total0": np.zeros(G, dtype=np.int32), "task_forbid": forbid, "task_need": np.full(max(T, 1), -1, dtype=np.int32),
        "task_contrib": forbid.copy(), "task_kind": np.full(max(T, 1), -1, dtype=np.int32),
        "node_kind_count0": np.zeros((1, max(N, 1)), dtype=np.int32), "kind_unbound": np.zeros(1, dtype=np.uint8),
        "task_weight_off": np.zeros(T + 1, dtype=np.uint32), "weight_kind": np.zeros(1, dtype=np.int32),
        "weight_keyset": np.zeros(1, dtype=np.int32), "weight_value": np.zeros(1, dtype=np.int64),
    }
    if G > 64:
        both = abi.KB_XGROUP_FORBID | abi.KB_XGROUP_CONTRIB
        hi_lab = lab_of[:T] >= 32
        cnt = np.where(hi_lab, 2, 0)
        s.pod_affinity["task_xgroup_off"] = np.concatenate([[0], np.cumsum(cnt)]).astype(np.uint32)
        labs = lab_of[:T][hi_lab]
        x = np.stack([((2 * labs) << 2) | both, ((2 * labs + 1) << 2) | both], axis=1).reshape(-1)
        s.pod_affinity["task_xgroup"] = x.astype(np.uint32) if x.size else np.zeros(1, dtype=np.uint32)
    s.meta["spread_tasks"] = int((lab_of[:T] >= 0).sum()) if T else 0
    s.invalidate()
    return s


def add_running_members(s: Snapshot, run: dict, frac: float = 0.1, labels: int = 8, seed: int = 13) -> dict:
    """After add_host_spread: makes `frac` of the Running tasks `run` (running_of) replicas of the spread Deployments — each carries
    app=<L> and the label's required anti-affinity term, so it is a member of both groups of label L (2L, 2L + 1).  Updates
    group_count0 / group_total0 of the snapshot and KB_RUNNING_AFF_MEMBER of `run` in place, and returns the per-task group lists
    (kb_running.aff_group_off / aff_group) in the format builder.flatten emits under meta["running_aff_groups"]."""
    rng = np.random.Generator(np.random.PCG64(seed))
    pa, N = s.pod_affinity, s.N
    n = len(run["node"])
    lab = np.where(rng.random(n) < frac, rng.integers(0, labels, size=n), -1)
    off = np.zeros(n + 1, dtype=np.uint32)
    groups = []
    for i in range(n):
        if lab[i] >= 0:
            g = [2 * int(lab[i]), 2 * int(lab[i]) + 1]
            groups += g
            for x in g:
                pa["group_count0"][x * N + int(run["node"][i])] += 1
                pa["group_total0"][x] += 1
            run["flags"][i] |= abi.KB_RUNNING_AFF_MEMBER
        off[i + 1] = len(groups)
    s.meta["member_tasks"] = int((lab >= 0).sum())
    s.invalidate()
    return {"aff_group_off": off, "aff_group": np.array(groups, dtype=np.uint32)}


def add_node_pref(s: Snapshot, frac: float = 0.3, seed: int = 11) -> Snapshot:
    """Gives `frac` of the PodGroups the preferred zone affinity Helm charts and operators commonly set: every pod of the group carries
    1-3 nodeAffinity.preferredDuringSchedulingIgnoredDuringExecution terms {zone In [z]} with weights from {1, 10, 50, 100}.  The zones
    are the label atoms `generate` sets (word 0, bits 0-2).  Fills KB_TASK_HAS_PREFERRED_NODE_AFFINITY and task_n_pref_terms /
    task_pref_terms / task_pref_weights exactly as builder.flatten would for such pods."""
    rng = np.random.Generator(np.random.PCG64(seed))
    for j in range(s.J):
        lo, hi = int(s.job_task_off[j]), int(s.job_task_off[j + 1])
        if hi == lo or rng.random() >= frac:
            continue
        nt = int(rng.integers(1, 4))
        zones = rng.integers(0, 3, size=nt)
        weights = rng.choice([1, 10, 50, 100], size=nt)
        s.task_flags[lo:hi] |= abi.KB_TASK_HAS_PREFERRED_NODE_AFFINITY
        s.task_n_pref_terms[lo:hi] = nt
        s.task_pref_terms[:, :, lo:hi] = 0
        s.task_pref_weights[:, lo:hi] = 0
        for p in range(nt):
            s.task_pref_terms[p, 0, lo:hi] = np.uint64(1) << np.uint64(zones[p])
            s.task_pref_weights[p, lo:hi] = weights[p]
    s.meta["pref_tasks"] = int((s.task_n_pref_terms != 0).sum())
    s.invalidate()
    return s


def add_pod_pref(s: Snapshot, frac: float = 0.15, labels: int = 8, seed: int = 17) -> Snapshot:
    """Gives `frac` of the PodGroups the soft spread many Helm charts set by default: every pod of the group carries app=<L> (L = one
    of `labels` values) and podAntiAffinity.preferredDuringSchedulingIgnoredDuringExecution {app=<L>, topologyKey
    kubernetes.io/hostname} with a weight w from {1, 10, 50, 100}.  Fills kb_pod_affinity (include/kbgpu.h) exactly as
    builder.flatten_pod_affinity would for such pods (one namespace, no placed pod carries the label or terms): no counter group;
    one pod kind per distinct (L, w), numbered in task order, unbound (a pod placed in the session keeps Spec.NodeName ""); one key
    set (hostname: a domain per node); the weight list of a pod of (L, w) holds, per kind (L, w') in kind order, -(w + w') — its own
    term plus the symmetric one of the other pod.  The snapshot must not carry kb_pod_affinity yet."""
    assert s.pod_affinity is None, "add_pod_pref builds kb_pod_affinity from scratch"
    rng = np.random.Generator(np.random.PCG64(seed))
    T, N = s.T, s.N
    kinds: Dict[Tuple[int, int], int] = {}
    task_kind = np.full(max(T, 1), -1, dtype=np.int32)
    for j in range(s.J):
        lo, hi = int(s.job_task_off[j]), int(s.job_task_off[j + 1])
        if hi == lo or rng.random() >= frac:
            continue
        lw = (int(rng.integers(0, labels)), int(rng.choice([1, 10, 50, 100])))
        task_kind[lo:hi] = kinds.setdefault(lw, len(kinds))
        s.task_flags[lo:hi] |= abi.KB_TASK_HAS_POD_AFFINITY
    NK = len(kinds)
    of_kind = list(kinds.keys())
    wlist = [[(k, -(w + w2)) for k, (l2, w2) in enumerate(of_kind) if l2 == lab] for (lab, w) in of_kind]
    cnt = np.array([len(wlist[k]) if k >= 0 else 0 for k in task_kind[:T]], dtype=np.int64)
    w_off = np.concatenate([[0], np.cumsum(cnt)]).astype(np.uint32)
    wk = [k2 for k in task_kind[:T] if k >= 0 for (k2, _) in wlist[k]]
    wv = [v for k in task_kind[:T] if k >= 0 for (_, v) in wlist[k]]
    s.pod_affinity = {
        "n_keysets": 1, "n_groups": 0, "n_kinds": NK, "n_weights": len(wk), "first_unbound_node": -1,
        "node_domain": np.arange(max(N, 1), dtype=np.int32).reshape(1, -1), "keyset_domains": np.array([N], dtype=np.uint32),
        "group_keyset": np.zeros(1, dtype=np.uint32), "group_count0": np.zeros(1, dtype=np.int32),
        "group_total0": np.zeros(1, dtype=np.int32), "task_forbid": np.zeros(max(T, 1), dtype=np.uint64),
        "task_need": np.full(max(T, 1), -1, dtype=np.int32), "task_contrib": np.zeros(max(T, 1), dtype=np.uint64),
        "task_kind": task_kind, "node_kind_count0": np.zeros((max(1, NK), max(N, 1)), dtype=np.int32),
        "kind_unbound": np.ones(max(1, NK), dtype=np.uint8) if NK else np.zeros(1, dtype=np.uint8),
        "task_weight_off": w_off, "weight_kind": np.array(wk or [0], dtype=np.int32),
        "weight_keyset": np.zeros(max(1, len(wk)), dtype=np.int32), "weight_value": np.array(wv or [0], dtype=np.int64),
    }
    s.meta["pod_pref_tasks"] = int((task_kind[:T] >= 0).sum()) if T else 0
    s.meta["pod_pref_kinds"] = of_kind
    s.invalidate()
    return s


# ------------------------------------------------------------------------------------------------
# small randomised sessions for property / parity tests: every feature of the path at once
# ------------------------------------------------------------------------------------------------
def random_session(seed: int, tasks: int = 60, jobs: int = 8, nodes: int = 12, queues: int = 1,
                   min_member_frac: float = 1.0, hetero: float = 0.3, prio_levels: int = 3,
                   oversub: float = 1.3, R: int = 3, W: int = 2, be_frac: float = 0.05, be_variants: bool = False) -> Snapshot:
    spec = SynthSpec(f"rand{seed}", tasks=tasks, jobs=jobs, nodes=nodes, queues=queues,
                     min_member_frac=min_member_frac, hetero_job_frac=hetero, prio_levels=prio_levels,
                     oversub=oversub, seed=seed, R=R, W=W)
    s = generate(spec)
    rng = np.random.Generator(np.random.PCG64(seed ^ 0x5EED))
    # sprinkle BestEffort (empty Resreq) tasks — allocate must skip them (allocate.go:113-118)
    if s.T:
        be = rng.random(s.T) < be_frac
        s.task_resreq[:, be] = 0
        s.task_initreq[:, be] = 0
        s.task_flags[be] |= abi.KB_TASK_BEST_EFFORT_QOS
        s.task_nz_cpu[be] = 100           # DefaultMilliCPURequest / DefaultMemoryRequest (non_zero.go:32-40)
        s.task_nz_mem[be] = 200 * 1024 * 1024
        if be_variants:
            # backfill's corner cases: requests below the IsEmpty epsilons (still "empty", but AddTask subtracts them),
            # and an init container that makes InitResreq non-empty while Resreq is empty (allocate skips the task AND
            # backfill leaves it alone, backfill.go:47 / :66-68)
            u = rng.random(s.T)
            tiny = be & (u < 0.3)
            s.task_resreq[0, tiny] = 5.0
            s.task_initreq[0, tiny] = 5.0
            s.task_flags[tiny] &= ~np.uint32(abi.KB_TASK_BEST_EFFORT_QOS)
            s.task_nz_cpu[tiny] = 5
            init = be & (u > 0.8)
            s.task_initreq[0, init] = 500.0
    return s
