"""Seeded sessions whose deciding nodes sit where the kernels' launch geometry splits the node table, built at array level
(Snapshot), so that clusters of 200 000 nodes take a second to build.

`Geometry` restates the launch geometry of the device for a GPU of `sm` SMs (the code it restates is named at each rule):
  scan       kb_build.h scan_tpi + build_session: tile groups of tpi tiles, grid = min(groups, sm - 1) CTAs, group g in
             iteration g // grid of CTA g % grid (scan_phase's double-buffered TMA loop, kb_kernels.cuh)
  pipeline   kb_build.h build_session: tpc = ceil(NT / (sm - 1)) resident tiles per scanner CTA, pipe_S = ceil(NT / tpc) CTAs,
             cycle_kernel only while tpc <= max_tpc = (227 KiB - 8 KiB) / tile bytes (12 at R = 3 / W = 2), the per-visit kernels above
  evict      kb_evict_kernels.cu launch_evict: workers = min(ceil(N / 512), sm - 1), node n in pass n // (workers * 512)
  prepass    kb_engine.cu launch_visit_link: aff_prepass_kernel<0> / <2> on ag = min(ceil(N / 256), 4 sm) CTAs of 256 threads
             (a node per thread), <1> on ag1 = min(ceil(N / 8), 8 sm) CTAs of 8 warps (a node per warp)
  gang       kb_kernels.cuh gang_commit_kernel: a job's processed slots in chunks of 32 (one warp)
A boundary is the largest N at which a loop still runs one pass less; `boundary_ns()` puts N just below, at and just above each.

geometry_session() places, on purpose, the nodes that decide a class where a geometry bug would lose them: the only feasible
nodes of a class in the last tile / last pipeline CTA / a later scan, evict or prepass pass (a nodeSelector on a label only those
nodes carry; the nodes reserved that way carry a taint only their classes tolerate); a class whose two identical nodes are the first
and the last node, so its best node alternates between the first and the last pass; classes of exactly 31 / 32 / 33 / 40 feasible
nodes spread over the whole table with room for one pod each (the top-32 lists merged across iterations and CTAs, the lowest index
wins among identical nodes); PodGroups of 31, 32, 33, 64, 65 and 200 tasks whose minMember puts e* into each 32-slot chunk, with
best-effort tasks after them (backfill slots after the allocate slots).  Options add preferred node-affinity terms whose max-count
nodes are only in the last CTA / pass, an inter-pod weight list (the counter path) and a sparse Running table for reclaim / preempt
whose victims sit only in the evict workers' second pass.  coverage() reads, from the oracle's decisions, which passes, CTAs and
tiles the placements and evictions landed in."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from kube_batch_b200 import abi
from kube_batch_b200.snapshot import Snapshot

TILE = 128                # TILE_NODES
EVICT_THREADS = 512
AFF_THREADS = 256
GI = 1 << 30
NODE_CPU, NODE_MEM = 32000.0, 128.0 * GI
RESERVED = np.uint64(1 << 1)      # taint word 0 bit 1: nodes reserved for the classes that select them
ZONES = 3                         # label word 0 bits 0..2
REGION_BIT0 = 8                   # label word 0 bits 8.. : one per region


def tile_ncols(R, W):
    return 2 * R + 6 + 3 * W


def cdiv(a, b):
    return (a + b - 1) // b


@dataclass(frozen=True)
class Geometry:
    sm: int
    R: int = 3
    W: int = 2

    # ---- per-visit scan ----
    @property
    def tile_bytes(self):
        return tile_ncols(self.R, self.W) * TILE * 8

    @property
    def tpi(self):                                  # kb_build.h scan_tpi
        budget = (160 if self.R > 8 else 190) * 1024
        t = 4
        while t > 1 and 2 * t * self.tile_bytes > budget:
            t -= 1
        return t

    def n_groups(self, N):
        return cdiv(cdiv(N, TILE), self.tpi)

    def scan_grid(self, N):
        return max(1, min(self.n_groups(N), self.sm - 1))

    def scan_passes(self, N):
        return cdiv(self.n_groups(N), self.scan_grid(N))

    def scan_pass_of(self, N, n):
        return (n // TILE // self.tpi) // self.scan_grid(N)

    # ---- persistent pipeline ----
    @property
    def max_tpc(self):
        return (227 * 1024 - 8 * 1024) // self.tile_bytes if (self.R, self.W) == (3, 2) else 0

    def pipe_tpc(self, N):
        """Resident tiles per scanner CTA, or 0 when the session runs the per-visit kernels."""
        tpc = cdiv(cdiv(N, TILE), self.sm - 1)
        return tpc if 0 < tpc <= self.max_tpc else 0

    def pipe_S(self, N):
        tpc = self.pipe_tpc(N)
        return cdiv(cdiv(N, TILE), tpc) if tpc else 0

    def pipe_cta_of(self, N, n):
        return n // TILE // self.pipe_tpc(N)

    @property
    def pipe_limit(self):
        """Largest N on cycle_kernel: 12 tiles per scanner CTA at R = 3 / W = 2."""
        return self.max_tpc * (self.sm - 1) * TILE

    # ---- reclaim / preempt sweep ----
    def evict_workers(self, N):
        return max(1, min(cdiv(N, EVICT_THREADS), self.sm - 1))

    def evict_passes(self, N):
        return cdiv(N, self.evict_workers(N) * EVICT_THREADS)

    def evict_pass_of(self, N, n):
        return n // (self.evict_workers(N) * EVICT_THREADS)

    # ---- aff_prepass_kernel ----
    def ag(self, N):
        return max(1, min(cdiv(N, AFF_THREADS), 4 * self.sm))

    def ag1(self, N):
        return max(1, min(cdiv(N, AFF_THREADS // 32), 8 * self.sm))

    def prepass_passes(self, N):
        return cdiv(N, self.ag(N) * AFF_THREADS)

    def prepass1_passes(self, N):
        return cdiv(N, self.ag1(N) * (AFF_THREADS // 32))

    # ---- the boundaries: the largest N at which each loop runs one pass less ----
    def boundaries(self):
        s1 = self.sm - 1
        b = {"scan_pass2": s1 * self.tpi * TILE, "scan_pass3": 2 * s1 * self.tpi * TILE,
             "evict_pass2": s1 * EVICT_THREADS, "prepass1_pass2": 8 * self.sm * (AFF_THREADS // 32),
             "prepass_pass2": 4 * self.sm * AFF_THREADS}
        if self.max_tpc:
            for k in range(1, self.max_tpc):
                b[f"pipe_tpc{k + 1}"] = k * s1 * TILE
            b["pipe_fallback"] = self.pipe_limit
        return b

    def describe(self, N):
        d = dict(N=N, tiles=cdiv(N, TILE), scan_tpi=self.tpi, scan_grid=self.scan_grid(N), scan_passes=self.scan_passes(N),
                 evict_workers=self.evict_workers(N), evict_passes=self.evict_passes(N), prepass_passes=self.prepass_passes(N),
                 prepass1_passes=self.prepass1_passes(N))
        if self.max_tpc:
            d.update(pipe_tpc=self.pipe_tpc(N), pipe_S=self.pipe_S(N))
        return d


def boundary_ns(b):
    """Just below, at and just above boundary b: N % 128 in {127, 0, 1} when b is a multiple of 128."""
    return [b - 1, b, b + 1]


def device_sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ----------------------------------------------------------------------------------------------------------------------------
# regions: where a geometry bug would lose a node
# ----------------------------------------------------------------------------------------------------------------------------
def regions(geo: Geometry, N: int) -> dict:
    """name -> sorted node indices.  Every region is a few nodes at one place of the launch geometry."""
    last = [N - 2, N - 1]
    grid, tpi = geo.scan_grid(N), geo.tpi
    late_group = (geo.scan_passes(N) - 1) * grid                        # first group of the last scan pass
    r = {"first": [0, 1], "last": last, "late_scan": [min(N - 1, late_group * tpi * TILE + k) for k in (3, 200)],
         "alternate": [0, N - 1]}
    if geo.scan_passes(N) >= 3:
        r["scan_pass3"] = [min(N - 1, 2 * grid * tpi * TILE + 5)]
    if geo.pipe_tpc(N):
        first_of_last_cta = (geo.pipe_S(N) - 1) * geo.pipe_tpc(N) * TILE
        r["last_cta"] = [first_of_last_cta + 7, N - 3]
    if geo.evict_passes(N) >= 2:
        r["evict_pass2"] = [geo.evict_workers(N) * EVICT_THREADS + k for k in (2, 3, 600)]
    # a node of the prepass's first grid pass and the first node of its second: with the weight list on, pods of a bound kind on
    # the second one make it the class's best node, which it is only if that grid pass counts them
    if geo.prepass1_passes(N) >= 2:
        r["prepass1_pass2"] = [geo.ag1(N) * 8 - 5, geo.ag1(N) * 8]
    if geo.prepass_passes(N) >= 2:
        r["prepass_pass2"] = [geo.ag(N) * AFF_THREADS - 5, geo.ag(N) * AFF_THREADS]
    r = {k: sorted(set(int(x) for x in v if 0 <= x < N)) for k, v in r.items()}
    taken = set(n for v in r.values() for n in v)
    for k in (31, 32, 33, 40):          # disjoint from every other region: each node has room for one pod of its class only
        nodes = []
        for x in np.linspace(3 + k, N - 4 - k, k).astype(np.int64).tolist():
            while x in taken:
                x += 1
            taken.add(x)
            nodes.append(x)
        r[f"spread{k}"] = sorted(nodes)
    return r


# ----------------------------------------------------------------------------------------------------------------------------
# the session
# ----------------------------------------------------------------------------------------------------------------------------
GANG_JOBS = [(31, 31), (32, 32), (33, 33), (64, 40), (65, 65), (200, 100)]      # (tasks, minMember): e* in chunks 0, 0, 1, 1, 2, 3


def geometry_session(N: int, seed: int, geo: Geometry, pref: bool = False, pod_pref: bool = False, evict: bool = False,
                     background_jobs: int = 12, gang: bool = True):
    """One session on N nodes.  pref: preferred node-affinity terms whose max-count nodes are only in the last CTA / pass.
    pod_pref: an inter-pod weight list on some classes (the counter path: aff_prepass_kernel).  evict: the cluster is full, the
    usage belongs to queue 1, and a sparse Running table (snap.meta["running"]) puts the only victims in the evict workers' later
    pass; queue 0 reclaims, a high-priority job of queue 1 preempts.  The region of each class is in snap.meta["class_region"]."""
    rng = np.random.default_rng(seed)
    R, W = geo.R, geo.W
    reg = regions(geo, N)
    # the reserved classes: (region, tasks, minMember, request cpu milli, mem)
    jobs = []          # dicts: tasks, min, region (or None), prio, queue, be (best-effort tasks after the regular ones), req
    one_slot = {}      # region -> node room: 1 pod each
    for name in ("last", "late_scan", "scan_pass3", "last_cta", "prepass1_pass2", "prepass_pass2"):
        if name in reg:
            jobs.append(dict(tasks=3, min=1, region=name, req=(1000.0, 2.0 * GI), wlist=pod_pref and name.startswith("prepass")))
    jobs.append(dict(tasks=8, min=1, region="alternate", req=(4000.0, 16.0 * GI)))
    for k in (31, 32, 33, 40):
        jobs.append(dict(tasks=k + 2, min=1, region=f"spread{k}", req=(500.0, 1.0 * GI)))
        one_slot[f"spread{k}"] = True
    if gang:
        for i, (t, m) in enumerate(GANG_JOBS):
            jobs.append(dict(tasks=t, min=m, region=None, req=(250.0 * (1 + i % 2), 0.5 * GI), be=12 if i % 2 == 0 else 0))
    for _ in range(background_jobs):
        jobs.append(dict(tasks=int(rng.integers(2, 12)), min=int(rng.integers(0, 3)), region=None,
                         req=(float(rng.choice([500, 1000, 2000])), float(rng.choice([1, 2, 4])) * GI)))
    ev_reg = "evict_pass2" if "evict_pass2" in reg else "last"
    if evict:
        # queue 0: a job that reclaims from queue 1; queue 1: a high-priority job that preempts (plain, with preferred
        # node-affinity terms, with an inter-pod weight list)
        jobs.append(dict(tasks=2, min=1, region=ev_reg, req=(8000.0, 16.0 * GI), queue=0, prio=0))
        jobs.append(dict(tasks=2, min=1, region=ev_reg, req=(8000.0, 16.0 * GI), queue=1, prio=10))
        jobs.append(dict(tasks=1, min=1, region=ev_reg, req=(8000.0, 16.0 * GI), queue=1, prio=10, pref=True))
        jobs.append(dict(tasks=1, min=1, region=ev_reg, req=(8000.0, 16.0 * GI), queue=1, prio=10, wlist=True))
    Jp = len(jobs)
    fill_jobs = 2 if evict else 1                      # the Running pods' PodGroups (queue 1 when evict)
    J = Jp + fill_jobs
    Q = 2 if evict else 1
    per = np.array([j["tasks"] + j.get("be", 0) for j in jobs], dtype=np.int64)
    T = int(per.sum())
    s = Snapshot(R, W, N, T, J, Q)

    # ---- nodes: one shape, random usage in bricks of 1/64 ----
    alloc = np.zeros((R, N))
    alloc[0], alloc[1] = NODE_CPU, NODE_MEM
    s.node_allocatable[:] = alloc
    s.node_alloc_present[:] = 1 << 2
    s.node_alloc_cpu[:] = int(NODE_CPU)
    s.node_alloc_mem[:] = int(NODE_MEM)
    s.node_max_pods[:] = 110
    s.node_labels[0] = np.uint64(1) << (np.arange(N) % ZONES).astype(np.uint64)
    if evict:
        k = np.full(N, 64, dtype=np.int64)             # full: nothing fits anywhere unless a victim leaves
    else:
        k = rng.integers(8, 56, size=N)
    region_nodes = np.zeros(N, dtype=bool)
    for bit, (name, nodes) in enumerate(sorted(reg.items())):
        nodes = np.array(nodes, dtype=np.int64)
        s.node_labels[0, nodes] |= np.uint64(1) << np.uint64(REGION_BIT0 + bit)
        region_nodes[nodes] = True
    s.node_taints[0, region_nodes] |= RESERVED
    if not evict:
        k[region_nodes] = 16
        k[np.array(reg["alternate"])] = 16
    used = np.zeros((R, N))
    used[0], used[1] = alloc[0] / 64 * k, alloc[1] / 64 * k
    s.node_used[:] = used
    s.node_idle[:] = alloc - used
    s.node_pods[:] = k.astype(np.int32)
    for name in one_slot:
        s.node_max_pods[np.array(reg[name])] = k[np.array(reg[name])] + 1
    s.node_nz_cpu[:] = used[0].astype(np.int64)
    s.node_nz_mem[:] = used[1].astype(np.int64)

    # ---- jobs and tasks ----
    off = np.zeros(J + 1, dtype=np.int64)
    off[1:Jp + 1] = np.cumsum(per)
    off[Jp + 1:] = T
    s.job_task_off[:] = off.astype(np.uint32)
    s.task_res_present[:] = 1 << 2
    s.task_prio[:] = 1
    s.task_uid_rank[:] = rng.permutation(T).astype(np.uint32)
    region_bit = {name: bit for bit, name in enumerate(sorted(reg))}
    class_region = {}
    pref_tasks, wl_tasks = [], []
    for j, jd in enumerate(jobs):
        lo, hi = int(off[j]), int(off[j + 1])
        n_reg = jd["tasks"]
        c, m = jd["req"]
        s.task_resreq[0, lo:lo + n_reg], s.task_resreq[1, lo:lo + n_reg] = c, m
        s.task_nz_cpu[lo:hi], s.task_nz_mem[lo:hi] = int(c), int(m)
        if hi > lo + n_reg:                                           # best-effort tasks: backfill's
            s.task_flags[lo + n_reg:hi] |= abi.KB_TASK_BEST_EFFORT_QOS
            s.task_nz_cpu[lo + n_reg:hi], s.task_nz_mem[lo + n_reg:hi] = 100, 200 << 20
        s.task_initreq[:, lo:hi] = s.task_resreq[:, lo:hi]
        s.task_ctime[lo:hi] = j
        s.task_prio[lo:hi] = 1 + jd.get("prio", 0)
        if jd["region"] is not None:
            s.task_sel_req[0, lo:hi] = np.uint64(1) << np.uint64(REGION_BIT0 + region_bit[jd["region"]])
            s.task_tol[0, lo:hi] = RESERVED
            class_region[j] = jd["region"]
        if jd.get("pref"):
            pref_tasks += list(range(lo, hi))
        if jd.get("wlist"):
            wl_tasks += list(range(lo, hi))
        s.job_min_avail[j] = jd["min"]
        s.job_queue[j] = jd.get("queue", 0)
        s.job_prio[j] = jd.get("prio", 0)
    s.job_ctime[:] = np.arange(J)
    s.job_alloc0_present[:] = 1 << 2
    s.queue_weight[:] = 1
    s.queue_ctime[:] = np.arange(Q)
    # the Running usage belongs to the filler jobs (the last of them owns every pod the Running table lists)
    fill = np.arange(N) % fill_jobs
    for r in range(2):
        s.job_alloc0[r, Jp:] = np.bincount(fill, weights=used[r], minlength=fill_jobs)
    s.job_ready0[Jp:] = np.bincount(fill, weights=k, minlength=fill_jobs).astype(np.int32)
    s.job_min_avail[Jp:] = 1 if evict else s.job_ready0[Jp:]
    s.job_queue[Jp:] = 1 if evict else 0

    # ---- preferred node affinity: the max-count nodes only in the last CTA / pass ----
    if pref:
        far = "last_cta" if "last_cta" in reg else "late_scan"
        bit = np.uint64(1) << np.uint64(REGION_BIT0 + region_bit[far])
        for j, jd in enumerate(jobs):
            if jd["region"] is None and j % 2 == 0:
                pref_tasks += list(range(int(off[j]), int(off[j]) + jd["tasks"]))
        s.meta["pref_region"] = far
        pt = np.array(sorted(set(pref_tasks)), dtype=np.int64)
        s.task_flags[pt] |= abi.KB_TASK_HAS_PREFERRED_NODE_AFFINITY
        s.task_n_pref_terms[pt] = 2
        s.task_pref_terms[0, 0, pt] = bit                              # the reserved far nodes: weight 100
        s.task_pref_weights[0, pt] = 100
        s.task_pref_terms[1, 0, pt] = np.uint64(1)                     # zone a: weight 1
        s.task_pref_weights[1, pt] = 1
        # those far nodes must also be feasible for them: tolerate the reservation, and leave room
        s.task_tol[0, pt] |= RESERVED
    elif pref_tasks:
        pt = np.array(pref_tasks, dtype=np.int64)
        s.task_flags[pt] |= abi.KB_TASK_HAS_PREFERRED_NODE_AFFINITY
        s.task_n_pref_terms[pt] = 1
        s.task_pref_terms[0, 0, pt] = np.uint64(1) << np.uint64(REGION_BIT0 + region_bit[ev_reg])
        s.task_pref_weights[0, pt] = 50

    # ---- inter-pod weight list: two pod kinds.  Kind 0: the weighted pods themselves (app=l0, a soft anti-affinity to each other per
    # host), placed in the session, so unbound: the reference credits their weight to the first unbound pod's node.  Kind 1: pods
    # bound to the far node of each prepass region, app=l1, which the weighted pods prefer (weight 10): only counting the far node
    # in the prepass's later grid pass makes it the best node of its class ----
    if pod_pref:
        for j, jd in enumerate(jobs):
            if jd["region"] is None and j % 3 == 0:
                wl_tasks += list(range(int(off[j]), int(off[j]) + jd["tasks"]))
    if wl_tasks:
        wt = np.array(sorted(set(wl_tasks)), dtype=np.int64)
        task_kind = np.full(T, -1, dtype=np.int32)
        task_kind[wt] = 0
        s.task_flags[wt] |= abi.KB_TASK_HAS_POD_AFFINITY
        cnt = 2 * (task_kind >= 0).astype(np.int64)
        nw = int(cnt.sum())
        far = [reg[name][-1] for name in ("prepass1_pass2", "prepass_pass2") if name in reg]
        bound = np.repeat(np.array(far, dtype=np.int64), 2)                 # two bound pods on each far node
        kind_count0 = np.zeros((2, N), dtype=np.int32)
        np.add.at(kind_count0[1], bound, 1)
        s.pod_affinity = {
            "n_keysets": 1, "n_groups": 0, "n_kinds": 2, "n_weights": nw, "first_unbound_node": -1,
            "node_domain": np.arange(N, dtype=np.int32).reshape(1, -1), "keyset_domains": np.array([N], dtype=np.uint32),
            "group_keyset": np.zeros(1, dtype=np.uint32), "group_count0": np.zeros(1, dtype=np.int32),
            "group_total0": np.zeros(1, dtype=np.int32), "task_forbid": np.zeros(T, dtype=np.uint64),
            "task_need": np.full(T, -1, dtype=np.int32), "task_contrib": np.zeros(T, dtype=np.uint64),
            "task_kind": task_kind, "node_kind_count0": kind_count0, "kind_unbound": np.array([1, 0], dtype=np.uint8),
            "task_weight_off": np.concatenate([[0], np.cumsum(cnt)]).astype(np.uint32),
            "weight_kind": np.tile(np.array([0, 1], dtype=np.int32), nw // 2), "weight_keyset": np.zeros(nw, dtype=np.int32),
            "weight_value": np.tile(np.array([-20, 10], dtype=np.int64), nw // 2),
        }
        s.meta["pod_objects"] = _pod_objects(T, N, wt, bound, weight=10)
        s.meta["bound_kind_nodes"] = far

    # ---- the Running table: only the pods on the evict-region nodes (4 per node, each a quarter of the node) ----
    if evict:
        ev_nodes = np.array(reg[ev_reg] + reg["first"], dtype=np.int64)
        node = np.repeat(ev_nodes, 4).astype(np.uint32)
        n = len(node)
        resreq = np.zeros((R, n))
        resreq[0], resreq[1] = NODE_CPU / 4, NODE_MEM / 4
        # the first-pass nodes' pods are of high priority: a preemptor passes the predicate there but finds no victim
        prio = np.where(np.isin(node, reg["first"]), 100, 1).astype(np.int32)
        s.meta["running"] = {"node": node, "job": np.full(n, Jp + fill_jobs - 1, dtype=np.uint32), "resreq": resreq,
                             "res_present": np.full(n, 1 << 2, dtype=np.uint32), "prio": prio, "ctime": np.arange(n, dtype=np.int64),
                             "uid_rank": rng.permutation(n).astype(np.uint32), "flags": np.zeros(n, dtype=np.uint32)}
        # the filler job that owns them also owns those nodes' usage
        for r in range(2):
            s.job_alloc0[r, Jp:] = 0
        owner = np.where(np.isin(np.arange(N), ev_nodes), fill_jobs - 1, 0)
        for r in range(2):
            s.job_alloc0[r, Jp:] = np.bincount(owner, weights=used[r], minlength=fill_jobs)
        s.job_ready0[Jp:] = np.bincount(owner, weights=k, minlength=fill_jobs).astype(np.int32)
        s.job_min_avail[Jp:] = 1
    s.meta.update(class_region=class_region, regions=reg, pending_jobs=Jp, geometry=geo.describe(N))
    s.validate()
    return s


def _pod_objects(T, N, kind_tasks, bound_nodes, weight):
    """The oracle's interned pod objects (oracle/kbo.py kbo_pod_objects) of the weight list above: the pods kind_tasks carry
    app=l0, podAntiAffinity.preferred {weight, app In [l0]} and podAffinity.preferred {weight, app In [l1]}, both per hostname;
    one Running pod of a filler PodGroup on each entry of bound_nodes carries app=l1 and no terms; no other pod carries labels or
    terms."""
    ns, app, l0, l1 = 0, 1, 2, 3
    E = len(bound_nodes)
    has = np.zeros(T + E, dtype=np.uint8)
    has[kind_tasks] = 1
    labels = has.astype(np.int64)
    labels[T:] = 1
    lab_val = np.where(np.arange(T + E) < T, l0, l1)[labels > 0]
    terms = 2 * has.astype(np.int64)
    m = int(terms.sum())
    return {"P": T + E, "T": T, "pod_ns": np.full(T + E, ns, dtype=np.int32),
            "lab_off": np.concatenate([[0], np.cumsum(labels)]), "lab_key": np.full(len(lab_val), app), "lab_val": lab_val,
            "has_aff": has, "has_anti": has, "term_off": np.concatenate([[0], np.cumsum(terms)]),
            "term_kind": np.tile([2, 3], m // 2), "term_weight": np.full(m, weight), "term_topo": np.zeros(m), "term_nil": np.zeros(m),
            "term_ns_off": np.arange(m + 1), "term_ns": np.full(m, ns), "term_req_off": np.arange(m + 1),
            "req_key": np.full(m, app), "req_op": np.zeros(m), "req_val_off": np.arange(m + 1), "req_val": np.tile([l1, l0], m // 2),
            "pod_node": np.asarray(bound_nodes), "pod_listed": np.ones(E), "pod_in_tasks": np.ones(E), "pod_unbound": np.zeros(E),
            "n_topo": 1, "node_topo": (4 + np.arange(N, dtype=np.int32)).reshape(1, -1)}


# ----------------------------------------------------------------------------------------------------------------------------
# what the oracle reached
# ----------------------------------------------------------------------------------------------------------------------------
def far_node_placements(s: Snapshot, o) -> dict:
    """Prepass region -> tasks of its class the oracle placed on the region's far node (in the prepass's second grid pass), where
    the bound pods of the weighted kind sit: with pod_pref, the class goes there only if that pass counts them."""
    d = o.decisions
    out = {}
    for j, name in s.meta["class_region"].items():
        if name.startswith("prepass"):
            t = np.arange(int(s.job_task_off[j]), int(s.job_task_off[j + 1]))
            out[name] = int((d["node"][t] == s.meta["regions"][name][-1]).sum())
    return out


def coverage(s: Snapshot, o, geo: Geometry, evicted=None) -> dict:
    """From the oracle's decisions: the deepest scan / evict / prepass pass, pipeline CTA and tile a placement landed in, how
    many reserved classes placed every task they could on their region, and the gang chunks e* fell into."""
    N = s.N
    d = o.decisions
    placed = np.nonzero(d["node"] >= 0)[0]
    nodes = d["node"][placed].astype(np.int64)
    cov = dict(N=N, placements=len(placed))
    if len(nodes):
        cov["max_scan_pass"] = int((nodes // TILE // geo.tpi // geo.scan_grid(N)).max())
        cov["max_evict_pass"] = int((nodes // (geo.evict_workers(N) * EVICT_THREADS)).max())
        cov["max_prepass1_pass"] = int((nodes // (geo.ag1(N) * 8)).max())
        cov["max_prepass_pass"] = int((nodes // (geo.ag(N) * AFF_THREADS)).max())
        cov["last_tile_used"] = int((nodes // TILE == cdiv(N, TILE) - 1).any())
        if geo.pipe_tpc(N):
            cov["last_cta_used"] = int((nodes // TILE // geo.pipe_tpc(N) == geo.pipe_S(N) - 1).any())
    reg = s.meta["regions"]
    reached = {}
    for j, name in s.meta["class_region"].items():
        t = np.arange(int(s.job_task_off[j]), int(s.job_task_off[j + 1]))
        on = d["node"][t]
        ok = on[on >= 0]
        assert np.isin(ok, reg[name]).all(), (name, ok)
        reached[name] = reached.get(name, 0) + len(ok)
    cov["region_placements"] = reached
    # spread classes: every node of the region used once (31 / 32 / 33 / 40 candidates, one pod each)
    cov["spread_full"] = [k for k in (31, 32, 33, 40) if reached.get(f"spread{k}", 0) == len(reg[f"spread{k}"])]
    alt = reg["alternate"]
    j_alt = [j for j, n in s.meta["class_region"].items() if n == "alternate"][0]
    seq = d["node"][np.arange(int(s.job_task_off[j_alt]), int(s.job_task_off[j_alt + 1]))]
    steps = d["step"][np.arange(int(s.job_task_off[j_alt]), int(s.job_task_off[j_alt + 1]))]
    seq = seq[np.argsort(steps, kind="stable")]
    seq = seq[seq >= 0]
    cov["alternations"] = int((np.diff(seq) != 0).sum()) if len(seq) > 1 and set(seq.tolist()) == set(alt) else 0
    # gang: the chunk of e* (first dispatched slot = e*) of each large job, in processing (step) order
    chunks = []
    straddle = 0
    for j in range(s.meta["pending_jobs"]):
        lo, hi = int(s.job_task_off[j]), int(s.job_task_off[j + 1])
        if hi - lo < 31:
            continue
        t = np.arange(lo, hi)
        al = t[(d["kind"][t] == abi.KB_KIND_ALLOCATED) & (d["step"][t] != 0xFFFFFFFF)]
        if not len(al) or not d["dispatched"][al].any():
            continue
        al = al[np.argsort(d["step"][al], kind="stable")]
        estep = int(d["dispatch_step"][al[0]])
        estar = int(np.nonzero(d["step"][al] == estep)[0][0])
        chunks.append(estar // 32)
        # the backfill view's slots follow the allocate view's (gang_commit_kernel): best-effort tasks placed by backfill whose
        # slots cross a 32-slot boundary into a chunk after e*'s (slots counted from the task counts: every task is processed)
        be = t[(s.task_flags[t] & abi.KB_TASK_BEST_EFFORT_QOS) != 0]
        nb = int((d["node"][be] >= 0).sum())
        na = len(t) - len(be)
        if nb and (na + nb - 1) // 32 > na // 32 and (na + nb - 1) // 32 > estar // 32:
            straddle += 1
    cov["gang_estar_chunks"] = sorted(set(chunks))
    cov["backfill_slots_past_estar_chunk"] = straddle
    if evicted is not None:
        run = s.meta["running"]
        ev_nodes = run["node"][evicted].astype(np.int64)
        cov["evictions"] = int(evicted.sum())
        cov["max_evict_pass_of_victim"] = int((ev_nodes // (geo.evict_workers(N) * EVICT_THREADS)).max()) if len(ev_nodes) else -1
    return cov
