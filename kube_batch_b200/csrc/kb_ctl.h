// kb_ctl.h — device-resident session state and the (single-threaded) control plane of the
// allocate cycle: queue heap, job ordering, DRF / proportion bookkeeping and the visit state
// machine.  Host/device shared (KB_HD): the device runs it in lane 0 of the epilogue warp, the
// host uses the same functions to build the initial state, and tests/emu runs it on the CPU.
//
// It restates the *control flow* of actions/allocate/allocate.go:43-194 around the per-task work:
//   queues  util.PriorityQueue over ssn.QueueOrderFn — pushed ONCE PER JOB, so duplicates sit in the
//           heap with stale proportion shares; Go's container/heap is emulated bit-exactly.
//   jobs    util.PriorityQueue over ssn.JobOrderFn per queue — keys never go stale while a job is in the
//           heap (only the job being visited changes its DRF share / readiness), so "pop" == "minimum of a
//           strict total order": a list sorted once at load + a small pool of re-pushed jobs.
//   tasks   util.PriorityQueue over ssn.TaskOrderFn per job — static keys: sorted once at load.
#ifndef KB_CTL_H_
#define KB_CTL_H_

#include "kb_core.h"
#include "kb_aff.h"

namespace kb {

constexpr uint32_t KB_CHAIN_MAX = 4;        // classes one visit_chain_kernel launch can scan (cur_class + 3 predicted)
enum StopReason : uint32_t { STOP_RUN_DONE = 0, STOP_NOFIT = 1, STOP_YIELD = 2, STOP_RESCAN = 3 };

struct Ctl {
  uint32_t arrive;        // ticket counter of the scan CTAs
  uint32_t done;          // queues.Empty() reached (allocate.go:90-92)
  int32_t  cur_job;       // job being visited, -1 = none
  uint32_t cur_queue;
  uint32_t cur_class;     // class of the next run == class the next scan evaluates
  uint32_t cur_run;       // consecutive tasks of cur_class at the job's cursor
  uint32_t qheap_len;
  uint32_t step;          // next Allocate/Pipeline sequence number
  uint32_t tasks_processed, tasks_allocated, tasks_pipelined, visits, scans, rescans;
  uint32_t error;         // sticky: an invariant the reference would panic on
  unsigned long long pairs_logical, pairs_scanned, pairs_replayed;
  // phase timers of the LAST CTA of every launch, SM cycles (clock64), summed over the cycle
  unsigned long long cyc_scan, cyc_merge, cyc_replay, cyc_total, cyc_steps, cyc_ctl;
  // ---- scan / replay overlap (single GPU): launch k scans `scan_class` (the predicted class of the visit after the
  //      one being replayed) while the replayer CTA consumes `list` (produced by launch k-1).  The scanners skip the
  //      `excl` nodes — exactly the nodes the replayer may modify — and the replayer contributes their fresh keys
  //      for `scan_class` as `patch`, so the merged list is exact for the table state at the end of the launch.
  uint32_t scan_class;
  uint32_t n_excl;
  uint32_t list_class, list_valid;
  uint32_t patch_valid;
  uint32_t predictions, mispredictions;
  uint32_t xchg_epoch;     // peer-memory exchange: sequence number of the next scan (starts at 1; flags are zeroed per cycle)
  uint32_t bf_cursor;      // backfill view: next entry of the best-effort job list (DevSession.q_static)
  uint32_t bf_seeded;      // backfill view: step / counters were carried over from the allocate view
  // ---- chained visits (visit_chain_kernel): the next launch scans cur_class AND these predicted classes of the
  //      following visits in one pass over the table (~0u = none); see DevSession.kchain
  uint32_t chain[KB_CHAIN_MAX - 1];
  uint32_t chain_hits;     // visits replayed from a look-ahead list (no launch of their own)
  uint32_t excl[32];
  unsigned long long list[32];
  unsigned long long patch[32];
  // ---- persistent pipeline (cycle_kernel, kb_pipe.cuh): scan requests posted / of which the replayer had to wait for
  //      (no usable look-ahead list), candidate-chain extensions, lists consumed with a non-empty patch set, log entries patched
  uint32_t pipe_requests, pipe_urgent, pipe_extends, pipe_patched, pipe_patch_entries;
  uint32_t phantoms;      // backfill: tasks left Allocated on no node (ssn.Allocate sets the status before node.AddTask refuses, session.go:241-262)
  uint32_t pred_dead;     // ... with the predicates plugin enabled such a task makes InterPodAffinityMatches return an error for every later
                          // pair (PodLister lists it, GetNodeInfo("") fails: plugins/util/util.go:93-100, vendor/.../predicates.go:1381-1393):
                          // no node passes ssn.PredicateFn for the rest of the session
  unsigned long long cyc_wait;     // replayer cycles spent between posting the visit and the eval warps' results (list wait + eval)
  unsigned long long cyc_ring, cyc_plan;      // timing mode: hot-ring append + write-back command; planner
  // timing mode: pools of the next chain built ahead and taken / not fitting the visit / dropped because the chain went on
  uint32_t pipe_builds_used, pipe_builds_missed, pipe_builds_cancelled;
};

// ---- persistent pipeline: global mailboxes between the replayer CTA and the scanner CTAs (kb_pipe.cuh) ----
constexpr uint32_t PIPE_RING = 32;       // scan requests that can be in flight (request / list slots)
constexpr uint32_t PIPE_PATCH = 32;      // modification-log entries a look-ahead list may lag behind at its use
struct PipeG {
  uint32_t log_head;                     // modification-log entries published (release) by the replayer's writer warp
  uint32_t quit;                         // the cycle is over (or failed): scanners exit
  uint32_t error;
  uint32_t pad0[29];
  unsigned long long req[PIPE_RING][2];  // NCCL-LL style words (tag << 32 | payload): class, stamp; tag = seq + 1
  uint32_t ticket[PIPE_RING];            // scanner CTAs that delivered their list for the slot
  unsigned long long list[PIPE_RING][2 * KTOP];   // merged top-32 of a request: two LL words (low / high half) per key
  uint32_t ticket_pref[PIPE_RING];       // scanner CTAs that delivered pass 1 (preferred node affinity) for the slot
  unsigned long long pref[PIPE_RING][2]; // LL words of a request for a class with preferred terms: max count over the feasible nodes, nodes reaching it
};

struct DevSession {
  EvalConf cf;
  uint32_t N, T, J, Q, C;
  uint32_t NT;            // node tiles
  uint32_t ncols;         // u64 columns per tile
  uint32_t To;            // order slots (tasks that are not Resreq.IsEmpty())
  uint32_t gang_ready;    // gang registered JobReadyFn && EnabledJobReady
  uint32_t jobcmp[4];     // JobOrderFn chain (JobCmp), JOBCMP_NONE terminated
  uint32_t queue_order_proportion;
  uint32_t proportion_present, drf_present;
  uint32_t total_dims_mask;            // dims of drf totalResource.ResourceNames()
  double   total[KB_CLASS_R];          // sum of node Allocatable (drf.go:62-64), dims 0..KB_CLASS_R-1; the rest in total_hi
  // node table: NT tiles of [ncols][TILE_NODES] u64, see tile_col_* below
  uint64_t* tiles;
  double*   node_used;    // [R][N] bookkeeping only
  ClassRec* classes;      // [C]
  // tasks in TaskOrderFn order, grouped by job
  uint32_t* ord_task;     // [To] snapshot task index
  uint32_t* ord_class;    // [To]
  uint32_t* ord_run;      // [To] number of consecutive slots of the same class starting here (within the job)
  uint32_t* ord_peek;     // [To] first class != ord_class[i] later in the queue's static job order (prediction only), ~0u = none
  uint32_t overlap;       // 1: visit_kernel runs scanners + one replayer CTA concurrently (world == 1)
  uint32_t kchain;        // 1: one class per launch; 2 / 4: visit_chain_kernel scans that many classes per launch and replays
                          //    the following visits from the look-ahead lists (patched with the nodes modified meanwhile)
  uint32_t* ord_chain;    // [To][KB_CHAIN_MAX-1] classes of the next runs with a different class in the queue's static job order
  uint32_t backfill;      // 1: this view drives backfillAction.Execute (backfill.go:40-71): jobs in JobID order, a task without
                          //    a node does not end the job, no yield rule, no resource predicate (EvalConf.fit_mode 1)
  uint32_t* job_ord_off;  // [J+1]
  uint32_t* job_pos;      // [J] cursor into ord_* (pendingTasks[job.UID], allocate.go:110-126)
  // jobs
  int32_t*  job_min_avail;
  int32_t*  job_ready;    // ReadyTaskNum (job_info.go:383)
  double*   job_alloc;    // [R][J] drfAttr.allocated
  double*   job_share;    // drfAttr.share
  uint32_t* job_queue;
  int32_t*  job_prio;
  uint32_t* job_tb_rank;  // rank of (CreationTimestamp, UID): the JobOrderFn fallback (session_plugins.go:260-266)
  uint32_t* job_placed;   // tasks placed this cycle
  uint32_t* q_static;     // [J] job ids sorted by initial JobOrderFn key, grouped by queue
  uint32_t* q_static_off; // [Q+1]
  uint32_t* q_static_head;// [Q]
  uint32_t* dyn_jobs;     // [J] re-pushed jobs (allocate.go:186), CSR by queue like q_static: queue q's at [q_static_off[q], + q_dyn_len[q])
  uint32_t* q_dyn_len;    // [Q]
  // queues
  double*   q_deserved;   // [R][Q] proportion queueAttr.deserved
  uint32_t* q_deserved_present;
  double*   q_allocated;  // [R][Q]
  double*   q_share;
  int64_t*  q_ctime;
  uint32_t* qheap;        // [J] Go heap of queue ids
  kb_decision* dec;       // [T]
  uint64_t* cand;         // [grid][KTOP] per-CTA candidate lists of the current scan
  Ctl* ctl;
  // node-axis sharding (SURVEY.md §8e).  Every rank holds the full (replicated) tables; a rank SCANS tiles
  // [tile_lo, tile_hi) only, then the ranks all-gather their top-KTOP keys together with the candidates'
  // node records and every rank replays identically, so the replicas never diverge.
  uint32_t rank, world, tile_lo, tile_hi, nodes_per_rank;
  uint32_t tpi;           // node tiles a scan CTA stages per iteration (sized to shared memory)
  uint64_t* sendbuf;      // [xchg_u64(ncols)]: keys[32], then columns [ncols][32], then a flag row (word 0: backfill's "some node
                          // outside the list passes the plugin predicates" bit)
  uint64_t* recvbuf;      // [world] x the same
  // Peer-memory exchange (fused scan + exchange + replay, no NCCL inside the cycle): every rank exposes one region
  //   recv[2 parities][KB_MAX_WORLD][P2P_RANK_U64] u64, then flags[2][KB_MAX_WORLD] u64
  // through CUDA IPC; peer_base[r] is rank r's region as mapped into THIS process (peer_base[rank] is local).
  uint32_t p2p;
  uint64_t* peer_base[8];
  // persistent pipeline (one cooperative launch per cycle, kb_pipe.cuh): pipe_S scanner CTAs keep pipe_tpc node tiles each
  // resident in shared memory, the last CTA replays
  uint32_t pipe, pipe_S, pipe_tpc, pipe_pad;
  PipeG* pg;
  uint32_t* modlog;       // [To + 64] node ids in modification order (one entry per node a visit chain modified)
  uint64_t* pcand;        // [PIPE_RING][pipe_S][KTOP] per-CTA candidate lists of the requests in flight
  unsigned long long* ppref;   // [PIPE_RING][pipe_S] pass 1 of a scan for a class with preferred node-affinity terms: (max count << 32 | nodes reaching it) per CTA
  const ClassPref* class_pref; // [C] preferred terms of the classes, NULL when the session has none
  int32_t w_nodeaff;           // nodeaffinity.weight (nodeorder.go:111-117)
  uint32_t pad_pref;
  uint32_t* dbg;          // 64 progress words in mapped host memory (KB_PIPE_DEBUG=1; NULL otherwise): read by the host watchdog when a cycle hangs
  AffDev aff;             // inter-pod (anti)affinity tables and counters (kb_aff.h); aff.on == 0: the session carries none
  const double* total_hi; // [R - KB_CLASS_R] dims KB_CLASS_R.. of `total` (sessions with more dims than ClassRec holds), next to the
                          // wide class table in the immutable slab; read through total_of
};
// The class table as records of type CR (ClassRecT): ClassRec for a session that fits it, ClassRecWide for R > KB_CLASS_R,
// ClassRecAtoms for W > KB_CLASS_W; the preferred terms (class_pref) in the same word capacity
template <class CR>
KB_HD const CR* class_table(const DevSession& S) { return reinterpret_cast<const CR*>(S.classes); }
template <class CR>
KB_HD const ClassPrefOf<CR>* pref_table(const DevSession& S) { return reinterpret_cast<const ClassPrefOf<CR>*>(S.class_pref); }
// drf's totalResource in dimension k (k < R) of a session whose class capacity is RC
template <uint32_t RC = KB_CLASS_R>
KB_HD double total_of(const DevSession& S, const uint32_t k) {
  if (RC <= KB_CLASS_R) return S.total[k];
  return k < KB_CLASS_R ? S.total[k] : S.total_hi[k - KB_CLASS_R];
}
constexpr uint32_t KB_MAX_WORLD = 8;
constexpr uint32_t P2P_RANK_U64 = (2 + 2 * KB_NARROW_R + 6 + 3 * KB_NARROW_W) * 32;   // keys + widest record block + flag row (the
                                                                                      // sharded path takes R <= KB_NARROW_R, W <= KB_NARROW_W only)
constexpr uint32_t P2P_FLAG_OFF = 2 * KB_MAX_WORLD * P2P_RANK_U64;
constexpr size_t   P2P_REGION_BYTES = ((size_t)P2P_FLAG_OFF + 2 * KB_MAX_WORLD) * 8;

// one rank's block of the sharded exchange: keys, the candidates' records, one flag row
KB_HD uint32_t xchg_u64(uint32_t ncols) { return (2 + ncols) * 32; }

// ---- tile columns (u64 each, TILE_NODES entries per column) ----
KB_HD uint32_t tile_ncols(uint32_t R, uint32_t W) { return 2 * R + 6 + 3 * W; }
KB_HD uint32_t col_idle(uint32_t, uint32_t r) { return r; }
KB_HD uint32_t col_rel(uint32_t R, uint32_t r) { return R + r; }
KB_HD uint32_t col_alloc_cpu(uint32_t R) { return 2 * R; }
KB_HD uint32_t col_alloc_mem(uint32_t R) { return 2 * R + 1; }
KB_HD uint32_t col_nz_cpu(uint32_t R) { return 2 * R + 2; }
KB_HD uint32_t col_nz_mem(uint32_t R) { return 2 * R + 3; }
KB_HD uint32_t col_pods(uint32_t R) { return 2 * R + 4; }      // pods (low 32) | max_pods (high 32)
KB_HD uint32_t col_flags(uint32_t R) { return 2 * R + 5; }
KB_HD uint32_t col_labels(uint32_t R, uint32_t, uint32_t w) { return 2 * R + 6 + w; }
KB_HD uint32_t col_taints(uint32_t R, uint32_t W, uint32_t w) { return 2 * R + 6 + W + w; }
KB_HD uint32_t col_ports(uint32_t R, uint32_t W, uint32_t w) { return 2 * R + 6 + 2 * W + w; }
// The flags column holds KB_NODE_* in its low 32 bits (what flags() hands to the predicates) and, above them, whether the node's
// Idle / Releasing has no scalar map (Resource.ScalarResources == nil).  Resource.Sub leaves the scalars of such a vector alone
// (api/resource_info.go:143-160): a task may request up to 10 milli of a scalar the node does not list (LessEqual skips it), and
// its placement then takes nothing of that scalar.  Resource.Add of a request that names a scalar creates the map (:127-139).
// At load a vector has no map iff the node lists no scalar in Allocatable and every scalar of the vector is 0.
// While a vector has no map its scalars are 0, whatever the record holds: the replay's dense updates may take them below zero,
// which no LessEqual tells apart from 0 (a scalar request of 10 milli or less is skipped, a larger one fits neither).  TileAcc —
// the node state the engine reports, and the evictions' view — reads them as 0; evict_apply / pipeline_apply (kb_evict.h) zero
// them when an Add gives the vector its map.
constexpr uint64_t NODE_IDLE_NO_SCALARS = 1ull << 32;
constexpr uint64_t NODE_REL_NO_SCALARS = 1ull << 33;

KB_HD double u64_as_double(uint64_t u) {
#if defined(__CUDA_ARCH__)
  return __longlong_as_double((long long)u);
#else
  double d; __builtin_memcpy(&d, &u, 8); return d;
#endif
}
KB_HD uint64_t double_as_u64(double d) {
#if defined(__CUDA_ARCH__)
  return (uint64_t)__double_as_longlong(d);
#else
  uint64_t u; __builtin_memcpy(&u, &d, 8); return u;
#endif
}

// Node accessor over one tile column block (`base` = first u64 of the tile, `i` = node within tile).
// Works on a tile staged in shared memory by TMA and on the global copy alike.
struct TileAcc {
  const uint64_t* base; uint32_t i, R, W;
  KB_HD uint64_t col(uint32_t c) const { return base[c * TILE_NODES + i]; }
  KB_HD double idle(uint32_t r) const {          // a scalar of an Idle without a scalar map is 0 (NODE_IDLE_NO_SCALARS)
    return (r >= 2 && (col(col_flags(R)) & NODE_IDLE_NO_SCALARS)) ? 0.0 : u64_as_double(col(col_idle(R, r)));
  }
  KB_HD double rel(uint32_t r) const {
    return (r >= 2 && (col(col_flags(R)) & NODE_REL_NO_SCALARS)) ? 0.0 : u64_as_double(col(col_rel(R, r)));
  }
  KB_HD int64_t alloc_cpu() const { return (int64_t)col(col_alloc_cpu(R)); }
  KB_HD int64_t alloc_mem() const { return (int64_t)col(col_alloc_mem(R)); }
  KB_HD int64_t nz_cpu() const { return (int64_t)col(col_nz_cpu(R)); }
  KB_HD int64_t nz_mem() const { return (int64_t)col(col_nz_mem(R)); }
  KB_HD int32_t pods() const { return (int32_t)(uint32_t)(col(col_pods(R)) & 0xFFFFFFFFull); }
  KB_HD int32_t max_pods() const { return (int32_t)(uint32_t)(col(col_pods(R)) >> 32); }
  KB_HD uint32_t flags() const { return (uint32_t)col(col_flags(R)); }
  KB_HD uint64_t labels(uint32_t w) const { return col(col_labels(R, W, w)); }
  KB_HD uint64_t taints(uint32_t w) const { return col(col_taints(R, W, w)); }
  KB_HD uint64_t ports(uint32_t w) const { return col(col_ports(R, W, w)); }
};

// Resource.Add of a request naming a scalar on node record `t` (first column, TILE_NODES apart): the vectors in `which`
// (NODE_IDLE_NO_SCALARS / NODE_REL_NO_SCALARS) that had no scalar map get one, with every scalar at 0
KB_HD void set_scalar_maps(uint64_t* t, const uint32_t R, const uint64_t which) {
  uint64_t& fl = t[(size_t)col_flags(R) * TILE_NODES];
  for (uint32_t k = 2; k < R; ++k) {
    if (fl & which & NODE_IDLE_NO_SCALARS) t[(size_t)col_idle(R, k) * TILE_NODES] = double_as_u64(0.0);
    if (fl & which & NODE_REL_NO_SCALARS) t[(size_t)col_rel(R, k) * TILE_NODES] = double_as_u64(0.0);
  }
  fl &= ~which;
}

// ---------------------------------------------------------------------------------------------
// ordering
// ---------------------------------------------------------------------------------------------
KB_HD bool job_is_ready(const DevSession& S, uint32_t j) { return S.job_ready[j] >= S.job_min_avail[j]; }   // job_info.go:423-427
// ssn.JobReady (session_plugins.go:182-200): AND over enabled JobReadyFns; only gang registers one
KB_HD bool ssn_job_ready(const DevSession& S, uint32_t j) { return !S.gang_ready || job_is_ready(S, j); }

// ssn.JobOrderFn(l, r) (session_plugins.go:243-267) with priority.go:61-77, gang.go:96-119, drf.go:114-130
KB_HD bool job_before(const DevSession& S, uint32_t l, uint32_t r) {
  for (int i = 0; i < 4; ++i) {
    uint32_t c = S.jobcmp[i];
    if (c == JOBCMP_NONE) break;
    if (c == JOBCMP_PRIORITY) {
      int32_t lp = S.job_prio[l], rp = S.job_prio[r];
      if (lp > rp) return true;
      if (lp < rp) return false;
    } else if (c == JOBCMP_GANG) {
      bool lr = job_is_ready(S, l), rr = job_is_ready(S, r);
      if (lr != rr) return rr;            // not-ready first
    } else if (c == JOBCMP_DRF) {
      double ls = S.job_share[l], rs = S.job_share[r];
      if (ls < rs) return true;
      if (ls > rs) return false;          // NB `==` on floats decides "equal", like drf.go:121
    }
  }
  return S.job_tb_rank[l] < S.job_tb_rank[r];
}

// ssn.QueueOrderFn (session_plugins.go:270-295) with proportion.go:156-169
KB_HD bool queue_before(const DevSession& S, uint32_t l, uint32_t r) {
  if (S.queue_order_proportion) {
    double ls = S.q_share[l], rs = S.q_share[r];
    if (ls < rs) return true;
    if (ls > rs) return false;
  }
  int64_t lc = S.q_ctime[l], rc = S.q_ctime[r];
  if (lc == rc) return l < r;             // UID order == index order
  return lc < rc;
}

// Go container/heap (go1.13 src/container/heap/heap.go) over S.qheap
KB_HD void qheap_up(const DevSession& S, int j) {
  for (;;) {
    int i = (j - 1) / 2;
    if (i == j || !queue_before(S, S.qheap[j], S.qheap[i])) break;
    uint32_t t = S.qheap[i]; S.qheap[i] = S.qheap[j]; S.qheap[j] = t;
    j = i;
  }
}
KB_HD void qheap_down(const DevSession& S, int i0, int n) {
  int i = i0;
  for (;;) {
    int j1 = 2 * i + 1;
    if (j1 >= n || j1 < 0) break;
    int j = j1;
    int j2 = j1 + 1;
    if (j2 < n && queue_before(S, S.qheap[j2], S.qheap[j1])) j = j2;
    if (!queue_before(S, S.qheap[j], S.qheap[i])) break;
    uint32_t t = S.qheap[i]; S.qheap[i] = S.qheap[j]; S.qheap[j] = t;
    i = j;
  }
}
// With a single queue every heap entry is the same element: Push/Pop only move the length.
KB_HD void qheap_push(const DevSession& S, Ctl& c, uint32_t q) {
  if (S.Q == 1) { c.qheap_len += 1; return; }
  S.qheap[c.qheap_len] = q;
  c.qheap_len += 1;
  qheap_up(S, (int)c.qheap_len - 1);
}
KB_HD uint32_t qheap_pop(const DevSession& S, Ctl& c) {
  if (S.Q == 1) { c.qheap_len -= 1; return 0; }
  int n = (int)c.qheap_len - 1;
  uint32_t t = S.qheap[0]; S.qheap[0] = S.qheap[n]; S.qheap[n] = t;
  qheap_down(S, 0, n);
  c.qheap_len = (uint32_t)n;
  return S.qheap[n];
}

// ---------------------------------------------------------------------------------------------
// plugin bookkeeping
// ---------------------------------------------------------------------------------------------
// drf.calculateShare (drf.go:161-171)
template <uint32_t RC = KB_CLASS_R>
KB_HD void update_job_share(const DevSession& S, uint32_t j) {
  double res = 0;
  for (uint32_t k = 0; k < S.cf.R; ++k) {
    if (!((S.total_dims_mask >> k) & 1u)) continue;
    double sh = share_of(S.job_alloc[(size_t)k * S.J + j], total_of<RC>(S, k));
    if (sh > res) res = sh;
  }
  S.job_share[j] = res;
}
// proportion.updateShare (proportion.go:241-253)
KB_HD void update_queue_share(const DevSession& S, uint32_t q) {
  double res = 0;
  uint32_t present = S.q_deserved_present[q] | 3u;
  for (uint32_t k = 0; k < S.cf.R; ++k) {
    if (!((present >> k) & 1u)) continue;
    double sh = share_of(S.q_allocated[(size_t)k * S.Q + q], S.q_deserved[(size_t)k * S.Q + q]);
    if (sh > res) res = sh;
  }
  S.q_share[q] = res;
}
// ssn.Overused (session_plugins.go:165-179) -> proportion.go:198-209: deserved.LessEqual(allocated)
KB_HD bool queue_overused(const DevSession& S, uint32_t q) {
  if (!S.proportion_present) return false;
  const uint32_t Q = S.Q;
  return res_less_equal(S.cf.R, [&](uint32_t k) { return S.q_deserved[(size_t)k * Q + q]; },
                        [&](uint32_t k) { return S.q_allocated[(size_t)k * Q + q]; });
}

// AllocateFunc event handlers of drf (drf.go:136-144) and proportion (proportion.go:213-222) for one placed task
template <class CR>
KB_HD void on_allocate_event(const DevSession& S, uint32_t j, const CR& c) {
  const uint32_t q = S.job_queue[j];
  for (uint32_t k = 0; k < S.cf.R; ++k) {
    if (S.drf_present) S.job_alloc[(size_t)k * S.J + j] = KB_DADD(S.job_alloc[(size_t)k * S.J + j], c.resreq[k]);
    if (S.proportion_present) S.q_allocated[(size_t)k * S.Q + q] = KB_DADD(S.q_allocated[(size_t)k * S.Q + q], c.resreq[k]);
  }
}

// ---------------------------------------------------------------------------------------------
// visit state machine
// ---------------------------------------------------------------------------------------------
KB_HD void setup_run(const DevSession& S, Ctl& c) {
  const uint32_t pos = S.job_pos[(uint32_t)c.cur_job];
  c.cur_class = S.ord_class[pos];
  c.cur_run = S.ord_run[pos];
}

// jobs.Pop() for queue q: minimum of {head of the static sorted list} U {re-pushed jobs of q}.  A queue's re-pushed jobs came
// off its static list, so they fit in its q_static range; job_before is a strict total order, so the scan order does not matter.
KB_HD int32_t pick_job(const DevSession& S, uint32_t q) {
  int32_t best = -1;
  int best_dyn = -1;
  uint32_t h = S.q_static_head[q];
  if (h < S.q_static_off[q + 1]) best = (int32_t)S.q_static[h];
  uint32_t* dyn = S.dyn_jobs + S.q_static_off[q];
  const uint32_t nd = S.q_dyn_len[q];
  for (uint32_t i = 0; i < nd; ++i) {
    uint32_t j = dyn[i];
    if (best < 0 || job_before(S, j, (uint32_t)best)) { best = (int32_t)j; best_dyn = (int)i; }
  }
  if (best < 0) return -1;
  if (best_dyn >= 0) { dyn[best_dyn] = dyn[nd - 1]; S.q_dyn_len[q] = nd - 1; }
  else S.q_static_head[q] = h + 1;
  return best;
}
KB_HD bool queue_has_jobs(const DevSession& S, uint32_t q) {
  return S.q_static_head[q] < S.q_static_off[q + 1] || S.q_dyn_len[q] != 0;
}

// The outer `for {}` of allocate.go:89-193 from "queues.Pop()" until a job with tasks is found.
// BF: compile-time copy of DevSession.backfill (-1 = read it at run time); the allocate kernels are instantiated with 0
// so that the backfill branches cost them nothing.
template <int BF = -1>
KB_HD void select_next_visit(const DevSession& S, Ctl& c) {
  const bool bf = BF < 0 ? S.backfill != 0 : BF != 0;
  c.cur_job = -1;
  for (;;) {
    uint32_t q;
    int32_t j;
    if (bf) {
      // backfill.go:45-46: every job (JobID order, SURVEY.md §8c), its Pending tasks with an empty InitResreq in UID
      // order.  q_static holds the jobs that have such tasks; no queue heap, no overused check, no JobOrderFn.
      if (c.bf_cursor >= S.q_static_off[1]) { c.done = 1; return; }
      j = (int32_t)S.q_static[c.bf_cursor];
      c.bf_cursor += 1;
      q = S.job_queue[j];
      if (S.job_pos[j] >= S.job_ord_off[j + 1]) continue;       // an earlier action of the cycle placed all of its best-effort tasks
    } else {
      if (c.qheap_len == 0) { c.done = 1; return; }                      // :90-92
      q = qheap_pop(S, c);                                                // :94
      if (queue_overused(S, q)) continue;                                 // :95-98
      if (!queue_has_jobs(S, q)) continue;                                // :104-107
      j = pick_job(S, q);                                                 // :109
      c.visits += 1;
      if (S.job_pos[j] >= S.job_ord_off[j + 1]) {                         // tasks.Empty(): the for at :129 is skipped
        qheap_push(S, c, q);                                              // :192
        continue;
      }
    }
    c.cur_job = j;
    c.cur_queue = q;
    setup_run(S, c);
    return;
  }
}

// End of a launch: the classes the NEXT launch scans besides cur_class (prediction only — a miss costs nothing but the
// wasted look-ahead).
KB_HD void publish_chain(const DevSession& S, Ctl& c) {
  for (uint32_t k = 0; k + 1 < KB_CHAIN_MAX; ++k) c.chain[k] = 0xFFFFFFFFu;
  if (c.done || c.cur_job < 0 || S.kchain <= 1) return;
  const uint32_t s0 = S.job_pos[(uint32_t)c.cur_job];
  for (uint32_t k = 0; k + 1 < KB_CHAIN_MAX && k + 1 < S.kchain; ++k) c.chain[k] = S.ord_chain[(size_t)s0 * (KB_CHAIN_MAX - 1) + k];
}

// Called once a run stopped.  `placed` = tasks of the run that went through Allocate/Pipeline.
// shares_done: the caller already refreshed the job's drf share and the queue's proportion share (the replay warp does
// the divisions of all dimensions in parallel lanes).  RC: class capacity of the session (drf's totals past KB_CLASS_R, total_of)
template <int BF = -1, uint32_t RC = KB_CLASS_R>
KB_HD void after_run(const DevSession& S, Ctl& c, uint32_t reason, uint32_t placed, const bool shares_done = false) {
  const bool bf = BF < 0 ? S.backfill != 0 : BF != 0;
  const uint32_t j = (uint32_t)c.cur_job;
  if (placed && !shares_done) {
    if (S.drf_present) update_job_share<RC>(S, j);
    if (S.proportion_present) update_queue_share(S, S.job_queue[j]);
  }
  if (reason == STOP_RESCAN) { setup_run(S, c); return; }
  bool end_visit;
  if (reason == STOP_NOFIT) end_visit = bf ? (S.job_pos[j] >= S.job_ord_off[j + 1])   // backfill.go:50-65: next task
                                                   : true;                                    // :144-148 break, job not re-pushed
  else if (reason == STOP_YIELD) {                                      // :185-188
    const uint32_t q = S.job_queue[j];
    S.dyn_jobs[S.q_static_off[q] + S.q_dyn_len[q]] = j; S.q_dyn_len[q] += 1;
    end_visit = true;
  } else end_visit = S.job_pos[j] >= S.job_ord_off[j + 1];
  if (!end_visit) { setup_run(S, c); return; }
  if (!bf) qheap_push(S, c, c.cur_queue);                               // :192
  select_next_visit<BF>(S, c);
}

// ---------------------------------------------------------------------------------------------
// Continuing a cycle on ONE session (scheduler.go:88-101 runs the configured actions one after the other on the same
// *framework.Session): what an action's own set-up reads from the session as the PREVIOUS actions left it.
// Single-threaded (one device thread / the host / tests/emu); J is small next to the work of the actions themselves.
// ---------------------------------------------------------------------------------------------
// job.TaskStatusIndex[Pending] of view S: tasks an earlier action placed are moved to the front of their job's slot range
// (order of the others kept) and the cursor starts behind them; run lengths are rebuilt for the rest.
KB_HD void prep_task_lists(const DevSession& S) {
  for (uint32_t j = 0; j < S.J; ++j) {
    const uint32_t lo = S.job_ord_off[j], hi = S.job_ord_off[j + 1];
    uint32_t front = lo;
    for (uint32_t i = lo; i < hi; ++i) {
      const uint8_t k = S.dec[S.ord_task[i]].kind;
      if (k != KB_KIND_ALLOCATED && k != KB_KIND_PIPELINED) continue;
      const uint32_t t = S.ord_task[i], c = S.ord_class[i];
      for (uint32_t m = i; m > front; --m) { S.ord_task[m] = S.ord_task[m - 1]; S.ord_class[m] = S.ord_class[m - 1]; }
      S.ord_task[front] = t; S.ord_class[front] = c;
      front += 1;
    }
    if (front != lo)
      for (uint32_t i = hi; i-- > front;) S.ord_run[i] = (i + 1 < hi && S.ord_class[i + 1] == S.ord_class[i]) ? S.ord_run[i + 1] + 1 : 1;
    S.job_pos[j] = front;
  }
}

// allocateAction.Execute's own queues (allocate.go:47-65) on the CURRENT state: JobOrderFn keys may have moved since the
// per-queue lists were sorted at load (few do: insertion sort), the queue heap is refilled with one push per job, the
// first visit is selected.  `step0`: the session's next Allocate / Pipeline sequence number.
KB_HD void prep_allocate(const DevSession& S, Ctl& c, const uint32_t step0) {
  for (uint32_t q = 0; q < S.Q; ++q) {
    const uint32_t lo = S.q_static_off[q], hi = S.q_static_off[q + 1];
    for (uint32_t i = lo + 1; i < hi; ++i) {
      const uint32_t v = S.q_static[i];
      uint32_t k = i;
      while (k > lo && job_before(S, v, S.q_static[k - 1])) { S.q_static[k] = S.q_static[k - 1]; --k; }
      S.q_static[k] = v;
    }
    S.q_static_head[q] = lo;
    S.q_dyn_len[q] = 0;
  }
  const uint32_t xe = c.xchg_epoch;
  c.done = 0; c.cur_job = -1; c.qheap_len = 0; c.error = 0;
  c.step = step0;
  for (uint32_t j = 0; j < S.J; ++j) qheap_push(S, c, S.job_queue[j]);      // one push PER JOB (allocate.go:52)
  select_next_visit<0>(S, c);
  c.scan_class = c.cur_class;
  c.n_excl = 0; c.list_valid = 0; c.patch_valid = 0;
  c.xchg_epoch = xe ? xe : 1;
  publish_chain(S, c);
}

// backfillAction.Execute's set-up on the current state (backfill.go:45-47 walks ssn.Jobs and their Pending tasks afresh)
KB_HD void prep_backfill(const DevSession& Sbf, Ctl& cb, const uint32_t step0) {
  prep_task_lists(Sbf);
  cb.done = 0; cb.cur_job = -1; cb.bf_cursor = 0; cb.error = 0;
  cb.step = step0;
  cb.bf_seeded = 1;
  select_next_visit<1>(Sbf, cb);
  cb.scan_class = cb.cur_class;
  if (!cb.xchg_epoch) cb.xchg_epoch = 1;
}

}  // namespace kb
#endif  // KB_CTL_H_
