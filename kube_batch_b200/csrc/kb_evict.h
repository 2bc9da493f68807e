// kb_evict.h — the two evicting actions of the cycle, host/device shared (KB_HD):
//   reclaimAction.Execute   actions/reclaim/reclaim.go:41-193     (ssn.Evict immediately, ssn.Pipeline)
//   preemptAction.Execute   actions/preempt/preempt.go:43-270     (framework.Statement: Evict / Pipeline, Commit / Discard)
// with the victim selection of the session (framework/session_plugins.go:80-162) over the built-in plugins' filters
// (gang.go:70-94, priority.go:81-100, drf.go:84-110, proportion.go:171-196, conformance.go:41-63).
//
// Shape of the work: per PREEMPTOR task one pass over all nodes — ssn.PredicateFn (K1, the same eval_pair as allocate),
// for preempt also the node score (K2, util.PrioritizeNodes + util.SortNodes == arg-max of the packed key; a class with preferred
// node-affinity terms first takes one more pass over all nodes for NodeAffinityPriority's max count), and per node a
// short SERIAL walk over the node's Running tasks (the plugins' filters are order-dependent: drf / proportion subtract
// cumulatively) -> "first node in order whose victims cover InitResreq".  The node axis is data-parallel (one thread per
// node, block arg-max); the commit on the chosen node (evictions, Pipeline, Statement log) is serial.  The control flow
// (queue heap, job heaps with stale keys like Go's container/heap, Statement commit / discard) is written ONCE as plain
// nested loops that every thread of the block executes uniformly; only thread 0 writes, barriers in between (Exec policy).
// tests/emu instantiates the same code with a one-thread Exec on the CPU and checks it against the oracle.
#ifndef KB_EVICT_H_
#define KB_EVICT_H_

#include "kb_ctl.h"

namespace kb {

enum EvictFn : uint32_t { EVF_GANG = 1u, EVF_PRIORITY = 2u, EVF_DRF = 4u, EVF_PROPORTION = 8u, EVF_CONFORMANCE = 16u };
constexpr uint32_t KB_EVICT_MAXV = 256;            // victims one node can hand to one preemptor (Running tasks on a node)

struct EvictConf {
  uint32_t reclaim_fns;        // the filters of the FIRST tier that has any enabled reclaimableFn (later tiers can only
  uint32_t preempt_fns;        //   intersect an empty set: session_plugins.go:112-115); 0 = no plugin registered one
  uint32_t gang_pipelined;     // gang registered && EnabledJobPipelined (session_plugins.go:203-221)
  uint32_t task_order_priority;
};

struct Preemptor {
  uint32_t task, job, queue, cls;
  uint32_t mode;           // 0 reclaim: Running tasks of OTHER queues; 1 preempt between jobs: same queue, other job; 2 preempt in job
  double ls;               // drf: share of the preemptor's job with the preemptor added (drf.go:87-89)
};

struct EvictCtl {
  uint32_t error;              // 1: the reference would panic (Resource.Sub on insufficient resource), 2: victim overflow
  uint32_t step;               // next Pipeline sequence number
  uint32_t n_evicted;          // cache.Evict calls so far
  uint32_t n_pipelined;
  uint32_t tasks_processed;    // preemptor tasks popped
  uint32_t scans;              // node sweeps really executed (identical failing sweeps are skipped, see try_preemptor)
  uint32_t version;            // bumped by every state change (eviction / pipeline / undo)
  uint32_t n_ops;              // Statement.operations
  uint32_t qheap_len;
  uint32_t fail_valid, fail_cls, fail_mode, fail_key, fail_version;   // the last sweep that found no node
  unsigned long long pairs_logical;
  // device plumbing of the master / worker kernel (kb_evict_kernels.cu): sweep mailbox, arg-max slot, the preemptor being
  // swept and its class (written by the master thread before it posts the command)
  uint32_t cmd_seq, arrived, n_workers, pad0;
  uint32_t cls_valid, cls_id;      // class record currently in `cls`      // master -> workers: sweep command counter (~0u = exit); workers -> master: CTAs done
  uint32_t pass;                   // master -> workers: 1 = pass 1 of a preferred node-affinity class (max count), 0 = the sweep
  uint32_t pmax;                   // workers -> master (pass 1): max count; master -> workers (sweep): the normalisation max
  unsigned long long red;
  Preemptor pre;
  ClassRec cls;
};

// Device view of the evict path's own data (everything else — node tiles, job / queue accounting, classes — is the
// DevSession's).  Running tasks are stored CSR by node, inside a node in TaskInfo.UID order (SURVEY.md §8c rule: the
// reference iterates the Go map n.Tasks).
struct EvictDev {
  EvictConf ec;
  uint32_t n_run, Tall;
  const uint32_t* node_off;      // [N+1]
  const uint32_t* r_orig;        // [n] slot -> index in the caller's kb_running arrays
  const uint32_t* r_job;         // [n]
  const double*   r_resreq;      // [R][n]
  const uint32_t* r_present;     // [n] scalar presence of Resreq
  const int32_t*  r_prio;        // [n] TaskInfo.Priority
  const int64_t*  r_ctime;       // [n]
  const uint32_t* r_uid_rank;    // [n]
  const uint32_t* r_flags;       // [n] KB_RUNNING_CRITICAL
  const uint32_t* pt_task;       // [Tall] ALL Pending tasks of every job, per job in TaskOrderFn order
  const uint32_t* pt_off;        // [J+1]
  const uint32_t* task_class;    // [T]
  const uint32_t* task_present;  // [T] scalar presence of the pending task's Resreq
  const int32_t*  job_waiting0;  // [J] Pipelined tasks of the job at session open (kb_running.job_waiting0)
  // mutable
  uint8_t*  r_state;             // [n] 0 Running, 1 Releasing (evicted)
  uint32_t* pt_pos;              // [J] tasks popped from preemptorTasks[job]
  int32_t*  job_waiting;         // [J] Pipelined tasks (WaitingTaskNum, job_info.go:396-405)
  uint32_t* jheap;               // [J] job heaps of the queues (preemptorsMap), CSR by queue (S.q_static_off)
  uint32_t* jheap_len;           // [Q]
  uint32_t* qheap;               // [Q] reclaim's queue heap (each queue pushed once, reclaim.go:60-66)
  uint32_t* q_alloc_present;     // [Q] scalar presence of proportion's queueAttr.allocated
  uint32_t* evict_order;         // [n] by slot: order of the cache.Evict call, 0xFFFFFFFF = not evicted
  uint32_t* ops;                 // [n + Tall] Statement.operations: bit 31 = Pipeline(task), else Evict(slot)
  uint32_t* scratch;             // [KB_EVICT_MAXV] victims of the node being committed
  EvictCtl* ctl;
};

// ---- api.Resource on dense vectors + presence masks (only where nil-ness is observable: Less) ----
// Resource.Less (resource_info.go:226-265)
template <class LAcc, class RAcc>
KB_HD bool res_less(uint32_t R, LAcc l, uint32_t lp, RAcc r, uint32_t rp) {
  if (!(l(0) < r(0))) return false;
  if (!(l(1) < r(1))) return false;
  lp &= ~3u; rp &= ~3u;
  if (lp == 0) {
    if (rp != 0)
      for (uint32_t k = 2; k < R; ++k) if (((rp >> k) & 1u) && r(k) <= KB_MIN_MILLI_SCALAR) return false;
    return true;
  }
  if (rp == 0) return false;
  for (uint32_t k = 2; k < R; ++k) {
    if (!((lp >> k) & 1u)) continue;
    const double q = ((rp >> k) & 1u) ? r(k) : 0.0;
    if (!(l(k) < q)) return false;
  }
  return true;
}

// drf.calculateShare (drf.go:161-171) of an allocation vector
KB_HD double drf_share_of(const DevSession& S, const double* alloc) {
  double res = 0;
  for (uint32_t k = 0; k < S.cf.R; ++k) {
    if (!((S.total_dims_mask >> k) & 1u)) continue;
    const double sh = share_of(alloc[k], S.total[k]);
    if (sh > res) res = sh;
  }
  return res;
}

// job.TaskStatusIndex[Pending] membership: a task an earlier action of the cycle placed (ssn.Allocate / ssn.Pipeline) left it
KB_HD bool task_pending(const DevSession& S, uint32_t t) { const uint8_t k = S.dec[t].kind; return k != KB_KIND_ALLOCATED && k != KB_KIND_PIPELINED; }

KB_HD bool evict_candidate(const DevSession& S, const EvictDev& E, const Preemptor& P, uint32_t slot) {
  if (E.r_state[slot] != 0) return false;                       // "Ignore non running task" (reclaim.go:127, preempt.go:105)
  const uint32_t j = E.r_job[slot];
  const uint32_t q = S.job_queue[j];
  if (P.mode == 0) return q != P.queue;                          // reclaim.go:131-136
  if (P.mode == 1) return q == P.queue && j != P.job;            // preempt.go:109-115
  return j == P.job;                                             // preempt.go:156-158
}

// One candidate through the deciding tier's filters.  `lo` = first slot of the node: drf / proportion subtract the
// candidates BEFORE this one (same job / same queue) cumulatively, in list order, exactly like the cloned allocations map.
KB_HD bool evict_is_victim(const DevSession& S, const EvictDev& E, const Preemptor& P, const uint32_t fns, const uint32_t lo, const uint32_t slot, uint32_t* err) {
  const uint32_t R = S.cf.R, n = E.n_run;
  const uint32_t j = E.r_job[slot];
  bool v = true;
  if (fns & EVF_GANG) {                                          // gang.go:70-90
    const int32_t occupid = S.job_ready[j];
    v = v && (S.job_min_avail[j] <= occupid - 1 || S.job_min_avail[j] == 1);
  }
  if (fns & EVF_PRIORITY) v = v && !(S.job_prio[j] >= S.job_prio[P.job]);       // priority.go:81-100
  if (fns & EVF_CONFORMANCE) v = v && !(E.r_flags[slot] & 1u);                   // conformance.go:45-58
  if (fns & EVF_DRF) {                                           // drf.go:90-107
    double ralloc[KB_MAX_R];
    for (uint32_t k = 0; k < R; ++k) ralloc[k] = S.job_alloc[(size_t)k * S.J + j];
    for (uint32_t s2 = lo; s2 <= slot; ++s2) {
      if (E.r_job[s2] != j || !evict_candidate(S, E, P, s2)) continue;
      if (!res_less_equal(R, [&](uint32_t k) { return E.r_resreq[(size_t)k * n + s2]; }, [&](uint32_t k) { return ralloc[k]; })) { *err = 1; return false; }
      for (uint32_t k = 0; k < R; ++k) ralloc[k] = KB_DSUB(ralloc[k], E.r_resreq[(size_t)k * n + s2]);
    }
    const double rs = drf_share_of(S, ralloc);
    v = v && (P.ls < rs || KB_FABS(KB_DSUB(P.ls, rs)) <= 0.000001);
  }
  if (fns & EVF_PROPORTION) {                                    // proportion.go:171-196
    const uint32_t q = S.job_queue[j];
    double al[KB_MAX_R];
    for (uint32_t k = 0; k < R; ++k) al[k] = S.q_allocated[(size_t)k * S.Q + q];
    const uint32_t ap = E.q_alloc_present[q];
    bool mine = false;
    for (uint32_t s2 = lo; s2 <= slot; ++s2) {
      if (S.job_queue[E.r_job[s2]] != q || !evict_candidate(S, E, P, s2)) continue;
      auto rq = [&](uint32_t k) { return E.r_resreq[(size_t)k * n + s2]; };
      if (res_less(R, [&](uint32_t k) { return al[k]; }, ap, rq, E.r_present[s2])) { if (s2 == slot) mine = false; continue; }   // "not enough resource": skipped
      if (!res_less_equal(R, rq, [&](uint32_t k) { return al[k]; })) { *err = 1; return false; }
      for (uint32_t k = 0; k < R; ++k) al[k] = KB_DSUB(al[k], rq(k));
      if (s2 == slot) mine = res_less_equal(R, [&](uint32_t k) { return S.q_deserved[(size_t)k * S.Q + q]; }, [&](uint32_t k) { return al[k]; });
    }
    v = v && mine;
  }
  return v;
}

// The preferred node-affinity terms preempt's node order reads for this preemptor (util.PrioritizeNodes with NodeAffinityPriority,
// registered by nodeorder; the condition visit_kernel uses), nullptr when the score has no such term.  reclaim walks ssn.Nodes in
// order and never scores (reclaim.go:113-115).
KB_HD const ClassPref* evict_pref(const DevSession& S, const Preemptor& P) {
  return (P.mode != 0 && S.class_pref != nullptr && S.cf.nodeorder && S.class_pref[P.cls].n != 0) ? &S.class_pref[P.cls] : nullptr;
}

// Pass 1 for such a preemptor, per node: its NodeAffinityPriority count when the node passes ssn.PredicateFn, else 0.
// NormalizeReduce divides by the max count over util.PredicateNodes (preempt.go:180-189, reduce.go:28-63), i.e. over EVERY node
// that passes the predicates — also nodes without Running tasks or eligible victims, and full nodes (preempt never checks Idle) —
// so this runs on all nodes, not only on those evict_node_key gives a key.  The max starts at 0, so 0 stands for "not counted".
KB_HD uint32_t evict_pref_count(const DevSession& S, const ClassRec& c, const ClassPref& cp, const uint32_t node) {
  const size_t tile_u64 = (size_t)S.ncols * TILE_NODES;
  TileAcc acc{S.tiles + (size_t)(node / TILE_NODES) * tile_u64, node % TILE_NODES, S.cf.R, S.cf.W};
  bool pok = true;
  (void)eval_pair(S.cf, c, acc, node, nullptr, &pok);
  if (!pok) return 0;
  const int32_t cnt = pref_count(cp, acc, S.cf.W);
  return cnt > 0 ? (uint32_t)cnt : 0u;
}

// K1 (+K2 for preempt) + the victim walk of one node: packed key (score, node) if the node's victims cover InitResreq, else 0.
// cp / pmax: evict_pref and the max of evict_pref_count over all nodes (pass 1); the score gains 10 * count / pmax times
// nodeaffinity.weight (a negative weight is already folded into cf.score_bias).
KB_HD uint64_t evict_node_key(const DevSession& S, const EvictDev& E, const Preemptor& P, const ClassRec& c, const ClassPref* cp, const uint32_t pmax,
                              const uint32_t node, uint32_t* err) {
  const uint32_t R = S.cf.R, W = S.cf.W, n = E.n_run;
  const uint32_t lo = E.node_off[node], hi = E.node_off[node + 1];
  if (lo == hi) return 0;
  const size_t tile_u64 = (size_t)S.ncols * TILE_NODES;
  TileAcc acc{S.tiles + (size_t)(node / TILE_NODES) * tile_u64, node % TILE_NODES, R, W};
  bool pok = true;
  const uint64_t k0 = eval_pair(S.cf, c, acc, node, nullptr, &pok);       // ssn.PredicateFn alone decides here (reclaim.go:115, preempt.go:179)
  (void)k0;
  if (!pok) return 0;
  const uint32_t fns = P.mode == 0 ? E.ec.reclaim_fns : E.ec.preempt_fns;
  if (fns == 0) return 0;                                                  // no plugin registered a filter: victims == nil
  double all[KB_MAX_R];
  for (uint32_t k = 0; k < R; ++k) all[k] = 0.0;
  uint32_t nv = 0;
  for (uint32_t s = lo; s < hi; ++s) {
    if (!evict_candidate(S, E, P, s)) continue;
    if (!evict_is_victim(S, E, P, fns, lo, s, err)) continue;
    for (uint32_t k = 0; k < R; ++k) all[k] = KB_DADD(all[k], E.r_resreq[(size_t)k * n + s]);
    ++nv;
  }
  if (nv == 0) return 0;                                                   // reclaim.go:141-144 / validateVictims
  if (!res_less_equal(R, [&](uint32_t k) { return c.initreq[k]; }, [&](uint32_t k) { return all[k]; })) return 0;   // :147-154
  if (P.mode == 0) return pack_key(S.cf.score_bias, node);
  const uint64_t key = pack_key(node_score(S.cf, c, acc), node);          // util.SortNodes: best score first, node order among equals
  return cp ? add_pref_term(key, (int64_t)S.w_nodeaff, (int64_t)pref_count(*cp, acc, W), (int64_t)pmax) : key;
}

// ---- state changes (thread 0) ----
// Session.Evict / Statement.Evict without the cache call: UpdateTaskStatus(Releasing), node.UpdateTask, DeallocateFunc handlers
KB_HD void evict_apply(const DevSession& S, const EvictDev& E, const uint32_t node, const uint32_t slot, const bool undo) {
  const uint32_t R = S.cf.R, n = E.n_run;
  const uint32_t j = E.r_job[slot], q = S.job_queue[j];
  const size_t tile_u64 = (size_t)S.ncols * TILE_NODES;
  uint64_t* t = S.tiles + (size_t)(node / TILE_NODES) * tile_u64 + (node % TILE_NODES);
  E.r_state[slot] = undo ? 0 : 1;
  // KB_RUNNING_AFF_MEMBER: the victim leaves util.PodLister — the member bits of the node records (host-level inter-pod
  // anti-affinity as atoms, kb_build.h) would have to change with it.  They do not: the cycle's outcome is withheld (error 3).
  if (!undo && (E.r_flags[slot] & KB_RUNNING_AFF_MEMBER) && E.ctl->error == 0) E.ctl->error = 3;
  S.job_ready[j] += undo ? 1 : -1;                                         // Running counts as ready, Releasing does not (job_info.go:383-393)
  for (uint32_t k = 0; k < R; ++k) {
    const double r = E.r_resreq[(size_t)k * n + slot];
    double idle = u64_as_double(t[(size_t)col_idle(R, k) * TILE_NODES]);
    double rel = u64_as_double(t[(size_t)col_rel(R, k) * TILE_NODES]);
    double used = S.node_used[(size_t)k * S.N + node];
    // node.UpdateTask = RemoveTask (by the node's clone status) + AddTask (new status), node_info.go:172-259
    if (!undo) { idle = KB_DSUB(KB_DADD(idle, r), r); rel = KB_DADD(rel, r); }                 // Running -> Releasing
    else       { rel = KB_DSUB(rel, r); idle = KB_DSUB(KB_DADD(idle, r), r); }                 // Releasing -> Running
    used = KB_DADD(KB_DSUB(used, r), r);
    t[(size_t)col_idle(R, k) * TILE_NODES] = double_as_u64(idle);
    t[(size_t)col_rel(R, k) * TILE_NODES] = double_as_u64(rel);
    S.node_used[(size_t)k * S.N + node] = used;
    if (S.drf_present) S.job_alloc[(size_t)k * S.J + j] = undo ? KB_DADD(S.job_alloc[(size_t)k * S.J + j], r) : KB_DSUB(S.job_alloc[(size_t)k * S.J + j], r);
    if (S.proportion_present) S.q_allocated[(size_t)k * S.Q + q] = undo ? KB_DADD(S.q_allocated[(size_t)k * S.Q + q], r) : KB_DSUB(S.q_allocated[(size_t)k * S.Q + q], r);
  }
  if (S.proportion_present && undo) E.q_alloc_present[q] |= E.r_present[slot] & ~3u;
  if (S.drf_present) update_job_share(S, j);
  if (S.proportion_present) update_queue_share(S, q);
  E.ctl->version += 1;
}

// Session.Pipeline / Statement.Pipeline (and Statement.unpipeline): UpdateTaskStatus(Pipelined), node.AddTask, AllocateFunc handlers
KB_HD void pipeline_apply(const DevSession& S, const EvictDev& E, const Preemptor& P, const ClassRec& c, const uint32_t node, const bool undo) {
  const uint32_t R = S.cf.R, W = S.cf.W;
  const uint32_t j = P.job, q = P.queue;
  const size_t tile_u64 = (size_t)S.ncols * TILE_NODES;
  uint64_t* t = S.tiles + (size_t)(node / TILE_NODES) * tile_u64 + (node % TILE_NODES);
  E.job_waiting[j] += undo ? -1 : 1;
  for (uint32_t k = 0; k < R; ++k) {
    const double r = c.resreq[k];
    double rel = u64_as_double(t[(size_t)col_rel(R, k) * TILE_NODES]);
    rel = undo ? KB_DADD(rel, r) : KB_DSUB(rel, r);                        // node_info.go:190-192 / :228-229
    t[(size_t)col_rel(R, k) * TILE_NODES] = double_as_u64(rel);
    S.node_used[(size_t)k * S.N + node] = undo ? KB_DSUB(S.node_used[(size_t)k * S.N + node], r) : KB_DADD(S.node_used[(size_t)k * S.N + node], r);
    if (S.drf_present) S.job_alloc[(size_t)k * S.J + j] = undo ? KB_DSUB(S.job_alloc[(size_t)k * S.J + j], r) : KB_DADD(S.job_alloc[(size_t)k * S.J + j], r);
    if (S.proportion_present) S.q_allocated[(size_t)k * S.Q + q] = undo ? KB_DSUB(S.q_allocated[(size_t)k * S.Q + q], r) : KB_DADD(S.q_allocated[(size_t)k * S.Q + q], r);
  }
  if (S.proportion_present && !undo) E.q_alloc_present[q] |= E.task_present[P.task] & ~3u;
  t[(size_t)col_nz_cpu(R) * TILE_NODES] = (uint64_t)((int64_t)t[(size_t)col_nz_cpu(R) * TILE_NODES] + (undo ? -c.nz_cpu : c.nz_cpu));
  t[(size_t)col_nz_mem(R) * TILE_NODES] = (uint64_t)((int64_t)t[(size_t)col_nz_mem(R) * TILE_NODES] + (undo ? -c.nz_mem : c.nz_mem));
  t[(size_t)col_pods(R) * TILE_NODES] = undo ? t[(size_t)col_pods(R) * TILE_NODES] - 1ull : t[(size_t)col_pods(R) * TILE_NODES] + 1ull;
  for (uint32_t w = 0; w < W; ++w) {
    uint64_t& pw = t[(size_t)col_ports(R, W, w) * TILE_NODES];
    pw = undo ? (pw & ~c.port_own[w]) : (pw | c.port_own[w]);
  }
  if (S.drf_present) update_job_share(S, j);
  if (S.proportion_present) update_queue_share(S, q);
  kb_decision d;
  d.node = undo ? -1 : (int32_t)node;
  d.kind = undo ? (res_is_empty(R, [&](uint32_t k) { return c.resreq[k]; }) ? KB_KIND_SKIPPED : KB_KIND_NONE) : KB_KIND_PIPELINED;
  d.dispatched = 0; d.reserved = 0;
  d.step = undo ? 0xFFFFFFFFu : E.ctl->step;
  d.dispatch_step = 0xFFFFFFFFu;
  S.dec[P.task] = d;
  if (!undo) { E.ctl->step += 1; E.ctl->n_pipelined += 1; } else E.ctl->n_pipelined -= 1;
  E.ctl->version += 1;
}

// reverse of ssn.TaskOrderFn on Running tasks: the victims queue of preempt.go:210-215 pops the LOWEST priority first
KB_HD bool victim_before(const EvictDev& E, uint32_t a, uint32_t b) {
  if (E.ec.task_order_priority && E.r_prio[a] != E.r_prio[b]) return E.r_prio[a] < E.r_prio[b];
  if (E.r_ctime[a] != E.r_ctime[b]) return E.r_ctime[a] > E.r_ctime[b];
  return E.r_uid_rank[a] > E.r_uid_rank[b];
}

// The serial part on the chosen node (thread 0): victims -> evictions until InitResreq is covered -> Pipeline.
// stmt: log into Statement.operations (preempt) instead of recording the cache.Evict right away (reclaim).
KB_HD void evict_commit(const DevSession& S, const EvictDev& E, const Preemptor& P, const ClassRec& c, const uint32_t node, const bool stmt) {
  const uint32_t R = S.cf.R, n = E.n_run;
  EvictCtl& ctl = *E.ctl;
  const uint32_t lo = E.node_off[node], hi = E.node_off[node + 1];
  const uint32_t fns = P.mode == 0 ? E.ec.reclaim_fns : E.ec.preempt_fns;
  uint32_t nv = 0, err = 0;
  for (uint32_t s = lo; s < hi; ++s) {
    if (!evict_candidate(S, E, P, s) || !evict_is_victim(S, E, P, fns, lo, s, &err)) continue;
    if (nv == KB_EVICT_MAXV) { ctl.error = 2; return; }
    E.scratch[nv++] = s;
  }
  if (err) { ctl.error = err; return; }
  if (stmt)                                                        // heap pops under a strict total order == sorted order
    for (uint32_t i = 1; i < nv; ++i) {
      const uint32_t v = E.scratch[i];
      uint32_t k = i;
      while (k > 0 && victim_before(E, v, E.scratch[k - 1])) { E.scratch[k] = E.scratch[k - 1]; --k; }
      E.scratch[k] = v;
    }
  double got[KB_MAX_R];
  for (uint32_t k = 0; k < KB_MAX_R; ++k) got[k] = 0.0;
  for (uint32_t i = 0; i < nv; ++i) {
    const uint32_t s = E.scratch[i];
    evict_apply(S, E, node, s, false);
    if (stmt) E.ops[ctl.n_ops++] = s;
    else E.evict_order[s] = ctl.n_evicted++;
    for (uint32_t k = 0; k < R; ++k) got[k] = KB_DADD(got[k], E.r_resreq[(size_t)k * n + s]);
    if (res_less_equal(R, [&](uint32_t k) { return c.initreq[k]; }, [&](uint32_t k) { return got[k]; })) break;   // reclaim.go:167-169, preempt.go:228-230
  }
  if (res_less_equal(R, [&](uint32_t k) { return c.initreq[k]; }, [&](uint32_t k) { return got[k]; })) {
    // node.AddTask(Pipelined) subtracts from Releasing and panics when it is short (resource_info.go:143-160)
    const size_t tile_u64 = (size_t)S.ncols * TILE_NODES;
    TileAcc acc{S.tiles + (size_t)(node / TILE_NODES) * tile_u64, node % TILE_NODES, R, S.cf.W};
    if (!res_less_equal(R, [&](uint32_t k) { return c.resreq[k]; }, [&](uint32_t k) { return acc.rel(k); })) { ctl.error = 1; return; }
    pipeline_apply(S, E, P, c, node, false);
    if (stmt) E.ops[ctl.n_ops++] = 0x80000000u | P.task;
  }
}

// Statement.Commit (statement.go:206-217): the evictions reach the cache in operation order
KB_HD void stmt_commit(const EvictDev& E) {
  EvictCtl& ctl = *E.ctl;
  for (uint32_t i = 0; i < ctl.n_ops; ++i) if (!(E.ops[i] & 0x80000000u)) E.evict_order[E.ops[i]] = ctl.n_evicted++;
  ctl.n_ops = 0;
}

// Go container/heap over an array with a comparator on CURRENT state (keys may be stale, like in the reference)
template <class Less>
KB_HD void heap_up(uint32_t* h, int j, Less less) {
  for (;;) {
    const int i = (j - 1) / 2;
    if (i == j || !less(h[j], h[i])) break;
    const uint32_t t = h[i]; h[i] = h[j]; h[j] = t;
    j = i;
  }
}
template <class Less>
KB_HD void heap_down(uint32_t* h, int i0, int n, Less less) {
  int i = i0;
  for (;;) {
    const int j1 = 2 * i + 1;
    if (j1 >= n || j1 < 0) break;
    int j = j1;
    const int j2 = j1 + 1;
    if (j2 < n && less(h[j2], h[j1])) j = j2;
    if (!less(h[j], h[i])) break;
    const uint32_t t = h[i]; h[i] = h[j]; h[j] = t;
    i = j;
  }
}
template <class Less>
KB_HD void heap_push(uint32_t* h, uint32_t& len, uint32_t v, Less less) { h[len] = v; len += 1; heap_up(h, (int)len - 1, less); }
template <class Less>
KB_HD uint32_t heap_pop(uint32_t* h, uint32_t& len, Less less) {
  const int n = (int)len - 1;
  const uint32_t t = h[0]; h[0] = h[n]; h[n] = t;
  heap_down(h, 0, n, less);
  len = (uint32_t)n;
  return h[n];
}

// ssn.JobPipelined (session_plugins.go:203-221) with gang.go:126-129 / job_info.go:430-434
KB_HD bool ssn_job_pipelined(const DevSession& S, const EvictDev& E, uint32_t j) {
  if (!E.ec.gang_pipelined) return true;
  return E.job_waiting[j] + S.job_ready[j] >= S.job_min_avail[j];
}

// ---------------------------------------------------------------------------------------------
// Exec policy: how the block runs the uniform control code.  X must provide
//   tid(), nthreads(), sync(), bcast(uint32_t) (thread 0's value, with barriers), block_max(uint64_t), cls() (ClassRec& scratch
//   every thread can read after a sync), and pre() (Preemptor& likewise).
// ---------------------------------------------------------------------------------------------
struct CpuExec {
  ClassRec c; Preemptor p;
  KB_HD int tid() const { return 0; }
  KB_HD int nthreads() const { return 1; }
  KB_HD void sync() {}
  KB_HD uint32_t bcast(uint32_t v) { return v; }
  KB_HD uint64_t block_max(uint64_t v) { return v; }
  KB_HD bool jobs_scanned() const { return false; }
  KB_HD void clear_max() {}
  uint64_t sweep(const DevSession& S, const EvictDev& E, const Preemptor& P, const ClassRec& c) {      // the node axis, serially
    const ClassPref* cp = evict_pref(S, P);
    uint32_t pmax = 0;
    if (cp)                                                       // pass 1 (preferred terms only): the normalisation max, on the current records
      for (uint32_t n = 0; n < S.N; ++n) { const uint32_t v = evict_pref_count(S, c, *cp, n); pmax = v > pmax ? v : pmax; }
    uint64_t best = 0;
    uint32_t err = 0;
    for (uint32_t n = 0; n < S.N; ++n) { const uint64_t k = evict_node_key(S, E, P, c, cp, pmax, n, &err); best = k > best ? k : best; }
    if (err) E.ctl->error = err;
    return best;
  }
  KB_HD ClassRec& cls() { return c; }
  KB_HD Preemptor& pre() { return p; }
};

// Start of an evicting action (reclaim.go:47-81, preempt.go:47-75): the action's own queues are filled from the session as it
// is NOW — jobs in the canonical job order, Go container/heap pushes with the comparators on the current state; a job
// enters with the tasks it still has in TaskStatusIndex[Pending].  Thread 0 only (J pushes of O(log J)).
// WaitingTaskNum and the cursor on the first Pending task of job j, from the decision table as the earlier actions left it
KB_HD void evict_scan_job(const DevSession& S, const EvictDev& E, const uint32_t j) {
  int32_t w = E.job_waiting0[j];
  uint32_t first = 0xFFFFFFFFu;
  for (uint32_t i = E.pt_off[j]; i < E.pt_off[j + 1]; ++i) {
    const uint32_t t = E.pt_task[i];
    if (S.dec[t].kind == KB_KIND_PIPELINED) w += 1;                  // WaitingTaskNum (job_info.go:396-405)
    if (first == 0xFFFFFFFFu && task_pending(S, t)) first = i - E.pt_off[j];
  }
  E.job_waiting[j] = w;
  E.pt_pos[j] = first == 0xFFFFFFFFu ? E.pt_off[j + 1] - E.pt_off[j] : first;   // cursor on the first Pending task
}

template <class X>
KB_HD void evict_init(X& x, const DevSession& S, const EvictDev& E) {
  EvictCtl& ctl = *E.ctl;
  x.sync();
  for (uint32_t j = (uint32_t)x.tid(); j < S.J && !x.jobs_scanned(); j += (uint32_t)x.nthreads()) {
    evict_scan_job(S, E, j);
  }
  x.sync();
  if (x.tid() == 0) {
    auto qless = [&](uint32_t l, uint32_t r) { return queue_before(S, l, r); };
    auto jless = [&](uint32_t l, uint32_t r) { return job_before(S, l, r); };
    ctl.qheap_len = 0; ctl.n_ops = 0; ctl.fail_valid = 0;
    for (uint32_t q = 0; q < S.Q; ++q) { E.jheap_len[q] = 0; E.scratch[q] = 0; }    // scratch doubles as queueMap (Q <= KB_MAX_Q <= KB_EVICT_MAXV)
    for (uint32_t j = 0; j < S.J; ++j) {
      const uint32_t q = S.job_queue[j];
      if (!E.scratch[q]) { E.scratch[q] = 1; heap_push(E.qheap, ctl.qheap_len, q, qless); }
      if (E.pt_pos[j] < E.pt_off[j + 1] - E.pt_off[j]) heap_push(E.jheap + S.q_static_off[q], E.jheap_len[q], j, jless);
    }
  }
  x.sync();
}

// tasks.Pop() of preemptorTasks[job] (thread 0): the next task of the job that is still Pending
KB_HD uint32_t evict_pop_task(const DevSession& S, const EvictDev& E, uint32_t job) {
  const uint32_t len = E.pt_off[job + 1] - E.pt_off[job];
  while (E.pt_pos[job] < len) {
    const uint32_t t = E.pt_task[E.pt_off[job] + E.pt_pos[job]];
    E.pt_pos[job] += 1;
    if (task_pending(S, t)) return t;
  }
  return 0xFFFFFFFFu;
}
KB_HD bool evict_has_task(const DevSession& S, const EvictDev& E, uint32_t job) {
  const uint32_t len = E.pt_off[job + 1] - E.pt_off[job];
  for (uint32_t i = E.pt_pos[job]; i < len; ++i) if (task_pending(S, E.pt_task[E.pt_off[job] + i])) return true;
  return false;
}

// One preemptor against all nodes; returns `assigned` (uniform across the block).
template <class X>
KB_HD bool try_preemptor(X& x, const DevSession& S, const EvictDev& E, const uint32_t task, const uint32_t job, const uint32_t mode, const bool stmt) {
  EvictCtl& ctl = *E.ctl;
  x.sync();
  if (x.tid() == 0) {
    Preemptor& P = x.pre();
    P.task = task; P.job = job; P.queue = S.job_queue[job]; P.cls = E.task_class[task]; P.mode = mode;
    if (!ctl.cls_valid || ctl.cls_id != P.cls) { x.cls() = S.classes[P.cls]; ctl.cls_id = P.cls; ctl.cls_valid = 1; }      // 408 B: only when it changes
    P.ls = 0.0;
    if (mode != 0 && (E.ec.preempt_fns & EVF_DRF)) {
      double la[KB_MAX_R];
      for (uint32_t k = 0; k < S.cf.R; ++k) la[k] = KB_DADD(S.job_alloc[(size_t)k * S.J + job], x.cls().resreq[k]);
      P.ls = drf_share_of(S, la);
    }
    ctl.tasks_processed += 1;
    ctl.pairs_logical += (unsigned long long)S.N;
    x.clear_max();
  }
  x.sync();
  const Preemptor& P = x.pre();
  const ClassRec& c = x.cls();
  // An identical sweep (same class, same filter, nothing changed since) that found no node finds none again: skip it.  This holds
  // with preferred node-affinity terms too: their scores only order the valid nodes, whether a valid node exists does not depend on them.
  const uint32_t fkey = mode == 0 ? P.queue : job;
  const bool known_fail = ctl.fail_valid && ctl.fail_cls == P.cls && ctl.fail_mode == mode && ctl.fail_key == fkey && ctl.fail_version == ctl.version;
  uint64_t best = 0;
  if (!known_fail) best = x.sweep(S, E, P, c);      // all nodes: K1 (+K2) + the victim walk, arg-max of the packed keys
  x.sync();
  if (x.tid() == 0) {
    if (!known_fail) ctl.scans += 1;
    if (best == 0) { ctl.fail_valid = 1; ctl.fail_cls = P.cls; ctl.fail_mode = mode; ctl.fail_key = fkey; ctl.fail_version = ctl.version; }
    else evict_commit(S, E, P, c, key_node(best), stmt);
  }
  x.sync();
  // assigned <=> the task was pipelined (evict_commit always reaches the Pipeline when the node was valid)
  return best != 0 && S.dec[task].kind == KB_KIND_PIPELINED;
}

// reclaimAction.Execute (reclaim.go:41-193)
template <class X>
KB_HD void run_reclaim(X& x, const DevSession& S, const EvictDev& E) {
  EvictCtl& ctl = *E.ctl;
  auto qless = [&](uint32_t l, uint32_t r) { return queue_before(S, l, r); };
  auto jless = [&](uint32_t l, uint32_t r) { return job_before(S, l, r); };
  evict_init(x, S, E);
  for (;;) {
    uint32_t task = 0xFFFFFFFFu, job = 0, q = 0, stop = 0;
    if (x.tid() == 0) {
      for (;;) {
        if (ctl.qheap_len == 0) { stop = 1; break; }                               // :85-87
        q = heap_pop(E.qheap, ctl.qheap_len, qless);                               // :92
        if (queue_overused(S, q)) continue;                                        // :93-96
        uint32_t* jh = E.jheap + S.q_static_off[q];
        if (E.jheap_len[q] == 0) continue;                                         // :99-101
        job = heap_pop(jh, E.jheap_len[q], jless);                                 // :102 (never pushed back)
        task = evict_pop_task(S, E, job);                                          // :106-109
        if (task == 0xFFFFFFFFu) continue;
        break;
      }
    }
    stop = x.bcast(stop);
    if (stop || ctl.error) break;
    task = x.bcast(task); job = x.bcast(job); q = x.bcast(q);
    const bool assigned = try_preemptor(x, S, E, task, job, 0u, false);
    if (x.tid() == 0 && assigned) heap_push(E.qheap, ctl.qheap_len, q, qless);     // :188-190
    x.sync();
  }
}

// preemptAction.Execute (preempt.go:43-167)
template <class X>
KB_HD void run_preempt(X& x, const DevSession& S, const EvictDev& E) {
  EvictCtl& ctl = *E.ctl;
  auto jless = [&](uint32_t l, uint32_t r) { return job_before(S, l, r); };
  auto pop_task = [&](uint32_t job) -> uint32_t { return evict_pop_task(S, E, job); };      // thread 0
  evict_init(x, S, E);
  for (uint32_t q = 0; q < S.Q && !ctl.error; ++q) {            // :78 `queues` is a Go map: ascending QueueID (SURVEY.md §8c)
    if (S.q_static_off[q + 1] == S.q_static_off[q]) continue;   // only queues that some job names
    uint32_t* jh = E.jheap + S.q_static_off[q];
    // ---- preemption between jobs within the queue (:80-136) ----
    for (;;) {
      uint32_t pj = 0xFFFFFFFFu;
      if (x.tid() == 0 && E.jheap_len[q] != 0) pj = heap_pop(jh, E.jheap_len[q], jless);      // :83-88
      pj = x.bcast(pj);
      if (pj == 0xFFFFFFFFu || ctl.error) break;
      bool assigned = false;
      for (;;) {                                                 // :92-125
        uint32_t t = 0xFFFFFFFFu;
        if (x.tid() == 0) t = pop_task(pj);
        t = x.bcast(t);
        if (t == 0xFFFFFFFFu) break;                             // :95-99
        if (try_preemptor(x, S, E, t, pj, 1u, true)) assigned = true;
        if (ctl.error) break;
        uint32_t pip = 0;
        if (x.tid() == 0) { pip = ssn_job_pipelined(S, E, pj) ? 1u : 0u; if (pip) stmt_commit(E); }   // :121-124
        pip = x.bcast(pip);
        if (pip) break;
      }
      if (ctl.error) break;
      uint32_t pip = 0;
      if (x.tid() == 0) {
        pip = ssn_job_pipelined(S, E, pj) ? 1u : 0u;
        if (!pip) {                                              // :128-131 stmt.Discard(): undo in reverse order
          for (uint32_t i = ctl.n_ops; i-- > 0;) {
            const uint32_t op = E.ops[i];
            if (op & 0x80000000u) {
              const uint32_t t = op & 0x7FFFFFFFu;
              Preemptor P; P.task = t; P.job = pj; P.queue = S.job_queue[pj]; P.cls = E.task_class[t]; P.mode = 1; P.ls = 0;
              pipeline_apply(S, E, P, S.classes[P.cls], (uint32_t)S.dec[t].node, true);
            } else {
              // the slot's node: binary search in node_off
              uint32_t lo = 0, hi = S.N;
              while (hi - lo > 1) { const uint32_t mid = (lo + hi) / 2; if (E.node_off[mid] <= op) lo = mid; else hi = mid; }
              evict_apply(S, E, lo, op, true);
            }
          }
          ctl.n_ops = 0;
        } else if (assigned) heap_push(jh, E.jheap_len[q], pj, jless);     // :133-135
      }
      x.sync();
      (void)pip;
    }
    // ---- preemption between tasks within a job (:138-166), over every job with Pending tasks ----
    for (uint32_t uj = 0; uj < S.J && !ctl.error; ++uj) {
      if (E.pt_off[uj + 1] == E.pt_off[uj]) continue;           // underRequest holds the jobs with Pending tasks
      for (;;) {
        uint32_t t = 0xFFFFFFFFu;
        if (x.tid() == 0) t = pop_task(uj);
        t = x.bcast(t);
        if (t == 0xFFFFFFFFu) break;                             // :141-144
        const bool assigned = try_preemptor(x, S, E, t, uj, 2u, true);
        if (x.tid() == 0) stmt_commit(E);                        // :161
        x.sync();
        if (!assigned || ctl.error) break;                       // :163-165
      }
    }
  }
}

}  // namespace kb
#endif  // KB_EVICT_H_
