// kb_kernels.cuh — sm_90a kernels of the allocate cycle.
//
//   visit_kernel          one launch = one SCAN of the node table for the class of the next run (K1 predicate bitmask +
//                         K2 fused score; node tiles staged into shared memory by TMA bulk copies, 16 warps = 4 tiles per
//                         iteration) -> per-warp / per-CTA top-32 candidate keys by bitonic networks (K3); the LAST CTA to
//                         finish (ticket) merges the lists, then warp 0 replays as many runs of that class as it can certify
//                         exactly (lane-owned candidates with a pre-evaluated next state, AddTask bookkeeping, gang stop
//                         rule) and runs the control plane (kb_ctl.h) to pick the next visit, while warp 1 prefetches the
//                         control plane's rows into L1.  The host only pumps a CUDA graph of launches until Ctl.done.
//                         Sharded node axis: the same kernel also performs the exchange over peer memory (NVLink stores +
//                         flags into CUDA-IPC mapped buffers) before the replay — scan, exchange and replay are ONE kernel.
//   replay_kernel         NCCL fallback of the sharded path: merge the all-gathered lists, same epilogue.
//   visit_overlap_kernel  opt-in: scanners run ahead on the predicted next class while one CTA replays (exclusion + patch).
//   gang_commit_kernel    K4: per-PodGroup inclusive prefix scan over the Allocated flags in processing order -> dispatched
//                         bit + dispatch step (framework/session.go:277-285).
//   matrix_kernel         full fit / score matrix for a task range (debug / parity, kb_predicate_score).
//   best_nodes_kernel     K1+K2+K3 over a task range x all nodes in ONE launch: per-task argmax via hardware warp reduce
//                         + one 64-bit atomicMax per warp (kb_best_nodes).
//
// No tensor cores anywhere: this is integer / FP64-compare work on an L2-resident table.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include "kb_ctl.h"

namespace kb {

constexpr int MATRIX_THREADS = TILE_NODES;         // matrix / best_nodes kernels: one node per thread, one tile per CTA
constexpr int SCAN_WARPS = 16;                     // visit_kernel: 16 warps = up to 4 node tiles in flight per iteration
constexpr int SCAN_THREADS = SCAN_WARPS * 32;
constexpr int MAX_TPI = SCAN_WARPS / 4;            // tiles per iteration (4 warps x 32 lanes cover one 128-node tile)
// widest node record of a session with class records of type CR (2R + 6 + 3W columns): 34 for the narrow instances, 82 for the
// wide ones, 70 for the wide-atom ones
template <class CR>
__host__ __device__ constexpr int max_cols() { return 2 * (int)CR::CAP + 6 + 3 * (int)CR::WCAP; }
constexpr unsigned FULL = 0xFFFFFFFFu;

// ---------------------------------------------------------------------------------------------
// TMA (1-D bulk copy) + mbarrier helpers — SASS: UBLKCP / SYNCS
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// programmatic dependent launch (PTX griddepcontrol): see visit_kernel
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  } while (!ok);
}

// max of a 64-bit key across the warp as two hardware 32-bit warp reductions (REDUX): high word first,
// then the low word among the lanes that hold the winning high word
__device__ __forceinline__ uint64_t warp_max_u64(uint64_t v) {
  const unsigned hi = (unsigned)(v >> 32), lo = (unsigned)v;
  const unsigned mhi = __reduce_max_sync(FULL, hi);
  const unsigned mlo = __reduce_max_sync(FULL, hi == mhi ? lo : 0u);
  return ((uint64_t)mhi << 32) | (uint64_t)mlo;
}

// Strided column accessor (shared-memory tile: stride TILE_NODES; dirty slots: stride DMAX)
struct ColAcc {
  const uint64_t* base; uint32_t i, stride, R, W;
  __device__ __forceinline__ uint64_t col(uint32_t c) const { return base[c * stride + i]; }
  __device__ __forceinline__ double idle(uint32_t r) const { return u64_as_double(col(col_idle(R, r))); }
  __device__ __forceinline__ double rel(uint32_t r) const { return u64_as_double(col(col_rel(R, r))); }
  __device__ __forceinline__ int64_t alloc_cpu() const { return (int64_t)col(col_alloc_cpu(R)); }
  __device__ __forceinline__ int64_t alloc_mem() const { return (int64_t)col(col_alloc_mem(R)); }
  __device__ __forceinline__ int64_t nz_cpu() const { return (int64_t)col(col_nz_cpu(R)); }
  __device__ __forceinline__ int64_t nz_mem() const { return (int64_t)col(col_nz_mem(R)); }
  __device__ __forceinline__ int32_t pods() const { return (int32_t)(uint32_t)(col(col_pods(R)) & 0xFFFFFFFFull); }
  __device__ __forceinline__ int32_t max_pods() const { return (int32_t)(uint32_t)(col(col_pods(R)) >> 32); }
  __device__ __forceinline__ uint32_t flags() const { return (uint32_t)col(col_flags(R)); }
  __device__ __forceinline__ uint64_t labels(uint32_t w) const { return col(col_labels(R, W, w)); }
  __device__ __forceinline__ uint64_t taints(uint32_t w) const { return col(col_taints(R, W, w)); }
  __device__ __forceinline__ uint64_t ports(uint32_t w) const { return col(col_ports(R, W, w)); }
};

// ---------------------------------------------------------------------------------------------
// Warp-level exact top-32 selection: bitonic networks over one key per lane (shuffles only).
// Lists are descending (lane 0 = best), 0-padded.  KTOP == 32 == warp size.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t warp_sort_desc(uint64_t v, int lane) {
#pragma unroll
  for (int k = 2; k <= 32; k <<= 1) {
#pragma unroll
    for (int j = k >> 1; j > 0; j >>= 1) {
      const uint64_t o = __shfl_xor_sync(FULL, v, j);
      const bool take_max = (((lane & k) == 0) == ((lane & j) == 0));
      v = take_max ? (o > v ? o : v) : (o < v ? o : v);
    }
  }
  return v;
}
// top-32 of the union of two descending lists, descending
__device__ __forceinline__ uint64_t warp_merge_top32(uint64_t a, uint64_t b, int lane) {
  const uint64_t br = __shfl_sync(FULL, b, 31 - lane);
  uint64_t v = a > br ? a : br;                  // bitonic sequence holding the 32 largest
#pragma unroll
  for (int j = 16; j > 0; j >>= 1) {
    const uint64_t o = __shfl_xor_sync(FULL, v, j);
    const bool take_max = (lane & j) == 0;
    v = take_max ? (o > v ? o : v) : (o < v ? o : v);
  }
  return v;
}


// CTA-level fold of the SCAN_WARPS per-warp lists into warp 0 (binary tree through shared memory).
// Every thread of the CTA must call it; returns the folded list in warp 0.
__device__ __forceinline__ uint64_t cta_fold_lists(uint64_t mine, uint64_t (*wlist)[KTOP], int warp, int lane) {
  // ping-pong between the two halves of wlist (rows [0,8) and [8,16)): the writers of round r+1 are readers of round r,
  // and they write the OTHER half, so one barrier per round is enough
  int flip = 0;
#pragma unroll
  for (int s = SCAN_WARPS / 2; s > 0; s >>= 1) {
    if (warp >= s && warp < 2 * s) wlist[flip * (SCAN_WARPS / 2) + (warp - s)][lane] = mine;
    __syncthreads();
    if (warp < s) mine = warp_merge_top32(mine, wlist[flip * (SCAN_WARPS / 2) + warp][lane], lane);
    flip ^= 1;
  }
  __syncthreads();      // callers reuse wlist right away
  return mine;
}

// forbidden counter groups >= 64 (ClassAff.xf_*) a scan CTA stages in shared memory: a class forbidden by more reads the rest from L2
constexpr uint32_t AFF_XF_SMEM = 128;

template <class CR = ClassRecNarrow>
struct VisitSmem {
  CR cls;
  ClassAff cls_aff;                          // inter-pod affinity record of the class (AFF instantiations only)
  AffX cls_xf[AFF_XF_SMEM];                  // the first AFF_XF_SMEM entries of its forbidden-group list (AFF instantiations only)
  ClassPrefOf<CR> cls_pref;                  // preferred node-affinity terms of the class (AFF instantiations, AffDev.has_pref)
  Ctl ctl;
  uint64_t keys[KTOP];                       // merged candidate list of the scan (K3 result)
  uint64_t wlist[SCAN_WARPS][KTOP];          // per-warp lists exchanged through shared memory
  uint64_t slot[2][max_cols<CR>()][32];      // candidate l: column c of state s at slot[s][c][l] (tile column scheme)
  uint64_t mbar[2];
  uint32_t is_last;
  uint32_t n_excl;
  uint32_t excl[32];                         // nodes the scanners skip (overlap mode)
  uint32_t sink;                             // keeps the shadow prefetch loads alive
  uint32_t pred_any;                         // backfill: some node of THIS CTA's tiles with key 0 passes ssn.PredicateFn (no Idle for Resreq)
  uint32_t pred_any_all;                     //   ... of any CTA / rank: what a task that finds no node needs to know (phantom Allocated)
  Ctl ctl2;                                  // replay_kernel's shadow warp reads its own copy
  // chained visits (visit_chain_kernel): nodes modified by the replays of this launch (no duplicates), the certification
  // floor of the list being replayed, and whether the last replay stopped for a rescan
  uint64_t chain_floor;
  uint32_t mod[KTOP * KB_CHAIN_MAX];
  uint32_t nmod;
  uint32_t nmod_prev;                        // sm.nmod before the last replay's appends
  uint32_t last_rescan;
  uint32_t chain_seq;                        // warp 0 -> shadow warp: a new chained visit is ready to be prefetched (~0u = stop)
  uint32_t lane_node[32], lane_which[32], lane_mod[32];   // the last replay's candidates: node, slot holding the current record, modified?
};

// ---------------------------------------------------------------------------------------------
// Exact replay + control plane, executed by ONE warp.  sm.keys holds the merged candidate list of the
// scan for class `cls_id` (sm.cls), sm.ctl a copy of the control block.  `rec_base`/`rec_stride` say
// where THIS lane's candidate record can be read (column c at rec_base[c * rec_stride]): the local node
// tiles on one GPU, the all-gathered records of the owning rank when the node axis is sharded.
// ---------------------------------------------------------------------------------------------
// Copies the control block back to global memory WITHOUT its first word (`arrive`, the ticket counter other CTAs may
// be incrementing right now).  One warp.
__device__ __forceinline__ void store_ctl(Ctl* g, const Ctl& c, int lane) {
  const uint32_t* src = reinterpret_cast<const uint32_t*>(&c);
  uint32_t* dst = reinterpret_cast<uint32_t*>(g);
  for (uint32_t i = 1 + lane; i < sizeof(Ctl) / 4; i += 32) dst[i] = src[i];
}

// `patch_class` != ~0u (overlap mode): after the replay, if the control plane's next visit has that class, every lane
// evaluates ITS candidate's current state for it and the sorted keys go to c.patch (see Ctl).  The caller stores c.
// CH = 1 (visit_chain_kernel): the floor comes from sm.chain_floor (a patched list's floor is not its 32nd key), the nodes
// this replay modified are appended to sm.mod and a rescan stop is reported in sm.last_rescan.
template <int BF, int CH = 0, int AFF = 0, class CR>
__device__ __forceinline__ void replay_epilogue(const DevSession& S, VisitSmem<CR>& sm, const int lane, const uint32_t cls_id,
                                                const uint64_t* rec_base, const uint32_t rec_stride, const uint32_t patch_class,
                                                const long long t_start, const long long t_scan) {
  // Lane l OWNS candidate l of the merged list: its node record lives in two shared-memory slots
  // (current state / state after one more placement of this class) and the lane keeps the packed key
  // of both.  A step is then a warp arg-max over the current keys; the chosen lane swaps to its
  // pre-evaluated next state.  eval_pair only runs in `refresh` rounds, for every lane whose look-ahead
  // is stale, all at once.  Exactness: nodes outside the list have keys < floor_key (the 32nd key of a
  // full list), so a pick is certified iff its key >= floor_key; otherwise the run stops for a rescan.
  Ctl& c = sm.ctl;
  const uint32_t R = S.cf.R, W = S.cf.W, ncols = S.ncols;
  if (lane == 0 && patch_class == 0xFFFFFFFFu) { c.scans += 1; c.pairs_scanned += (unsigned long long)S.N; }
  uint64_t cur_key = sm.keys[lane];
  const uint64_t floor_key = CH ? sm.chain_floor : sm.keys[KTOP - 1];
  const bool have = cur_key != 0;
  bool rescanned = false;
  const uint32_t my_node = key_node(cur_key);
  uint64_t* gt_mine = S.tiles + (size_t)(my_node / TILE_NODES) * (ncols * TILE_NODES) + (my_node % TILE_NODES);
  uint32_t which = 0;                 // slot holding my CURRENT state
  bool cur_fi = false, next_fi = false, next_valid = false, modified = false;
  uint64_t next_key = 0;
  if (have) {
    // the candidate's record: the first 18 columns (the whole record at R=3, W=2) as ONE batch of independent loads
    // = one L2 round trip; wider records finish in a loop
    constexpr uint32_t GATHER_UNROLL = 18;
    uint64_t tmp[GATHER_UNROLL];
#pragma unroll
    for (uint32_t cc = 0; cc < GATHER_UNROLL; ++cc) tmp[cc] = cc < ncols ? __ldcg(rec_base + (size_t)cc * rec_stride) : 0ull;
#pragma unroll
    for (uint32_t cc = 0; cc < GATHER_UNROLL; ++cc) if (cc < ncols) sm.slot[0][cc][lane] = tmp[cc];
    for (uint32_t cc = GATHER_UNROLL; cc < ncols; ++cc) sm.slot[0][cc][lane] = __ldcg(rec_base + (size_t)cc * rec_stride);
    ColAcc acc{&sm.slot[0][0][0], (uint32_t)lane, 32u, R, W};
    cur_fi = res_less_equal(R, [&](uint32_t k) { return sm.cls.initreq[k]; }, [&](uint32_t k) { return acc.idle(k); });
  }
  // look-ahead refresh: next state = current state + one placement (Allocate if InitResreq <= Idle else Pipeline)
  auto refresh = [&]() {
    const bool need = have && cur_key != 0 && !next_valid;
    const unsigned todo = __ballot_sync(FULL, need);
    if (need) {
      const uint64_t (*src)[32] = sm.slot[which];
      uint64_t (*dst)[32] = sm.slot[which ^ 1u];
      for (uint32_t cc = 0; cc < ncols; ++cc) dst[cc][lane] = src[cc][lane];
      const uint32_t base_col = cur_fi ? col_idle(R, 0) : col_rel(R, 0);
      for (uint32_t k = 0; k < R; ++k)
        dst[base_col + k][lane] = double_as_u64(KB_DSUB(u64_as_double(src[base_col + k][lane]), sm.cls.resreq[k]));
      dst[col_nz_cpu(R)][lane] = (uint64_t)((int64_t)src[col_nz_cpu(R)][lane] + sm.cls.nz_cpu);
      dst[col_nz_mem(R)][lane] = (uint64_t)((int64_t)src[col_nz_mem(R)][lane] + sm.cls.nz_mem);
      dst[col_pods(R)][lane] = src[col_pods(R)][lane] + 1ull;          // pods live in the low 32 bits
      for (uint32_t w = 0; w < W; ++w) dst[col_ports(R, W, w)][lane] = src[col_ports(R, W, w)][lane] | sm.cls.port_own[w] | (cur_fi ? sm.cls.aff_own[w] : 0ull);
      ColAcc acc{&dst[0][0], (uint32_t)lane, 32u, R, W};
      next_key = eval_pair(S.cf, sm.cls, acc, my_node, &next_fi);
      if (AFF && cur_fi && aff_self_blocks(S.aff, sm.cls_aff, S.N, my_node)) next_key = 0;   // one replica per host: the class's own pod, once ALLOCATED (a Pipelined
                                                                  // pod is not listed by util.PodLister), forbids the node (kb_aff.h)
      next_valid = true;
    }
    if (lane == 0) c.pairs_replayed += (unsigned long long)__popc(todo);
  };
  refresh();
  __syncwarp();
  const long long t_merge = clock64();

  uint32_t my_cnt = 0;        // placements on MY candidate (NodeInfo.Used delta = my_cnt x Resreq, applied at write-back)
  // inter-pod affinity (kb_aff.h): a class whose keys read counters that its own placement changes beyond the chosen node uses
  // its list for ONE placement — the placement can change the feasibility / score of every node of a topology domain
  const bool aff_rd = AFF && (aff_stop_each(sm.cls_aff, S.cf.nodeorder != 0) ||
                              (S.aff.has_pref && sm.cls_pref.n != 0 && S.cf.nodeorder != 0));      // the normalisation (max count) can move with every placement
  bool aff_stop = false;
  for (;;) {              // runs
    if (c.done || c.cur_class != cls_id || (AFF && aff_stop)) break;
    const uint32_t j = (uint32_t)c.cur_job;
    const uint32_t q = c.cur_queue;
    const uint32_t jend = S.job_ord_off[j + 1];
    uint32_t run_left = c.cur_run;
    uint32_t placed = 0, popped = 0, n_alloc = 0, n_phantom = 0;
    uint32_t reason = STOP_RUN_DONE;
    // job-level state of the run lives in registers: lane 0 keeps the counters, lane k < R keeps dimension k
    // of drfAttr.allocated / queueAttr.allocated; nothing but the decision store touches memory in a step
    const uint32_t pos0 = __shfl_sync(FULL, lane == 0 ? S.job_pos[j] : 0u, 0);
    int32_t ready = 0, min_avail = 0;
    if (lane == 0) { ready = S.job_ready[j]; min_avail = S.job_min_avail[j]; }
    ready = __shfl_sync(FULL, ready, 0); min_avail = __shfl_sync(FULL, min_avail, 0);
    double jalloc = 0.0, qalloc = 0.0, my_rq = 0.0;
    if (lane < R) {
      my_rq = sm.cls.resreq[lane];
      if (S.drf_present) jalloc = S.job_alloc[(size_t)lane * S.J + j];
      if (S.proportion_present) qalloc = S.q_allocated[(size_t)lane * S.Q + q];
    }
    const uint32_t step0 = c.step;
    uint32_t my_task = 0;       // lane l holds ord_task[window base + l]
    const long long t_run0 = clock64();
    while (run_left > 0) {      // steps: one pending task each
      const uint64_t best = warp_max_u64(cur_key);
      if (best < floor_key) { reason = STOP_RESCAN; break; }      // a node outside the list might win: cannot certify
      // pop the task (allocate.go:130); the ord_task window is refilled every 32 steps
      const uint32_t pos = pos0 + popped;
      if ((popped & 31u) == 0) my_task = (pos + lane < jend) ? S.ord_task[pos + lane] : 0u;
      const uint32_t task = __shfl_sync(FULL, my_task, popped & 31u);
      popped += 1;
      run_left -= 1;
      if (best == 0) {                                             // allocate.go:144-148
        if (BF) {
          // backfill.go:53-63 calls ssn.Allocate on every node that passes ssn.PredicateFn; ssn.Allocate moves the task to
          // Allocated BEFORE node.AddTask checks Resreq <= Idle (session.go:241-262).  No node took the task: if any node
          // passes the predicates the reference leaves it Allocated on no node (it counts towards JobReady from now on).
          // Nodes outside the list are unmodified since the scan (their bit is pred_any_all); candidates are re-checked.
          bool pk = false;
          if (have) {
            ColAcc acc{&sm.slot[which][0][0], (uint32_t)lane, 32u, R, W};
            eval_pair(S.cf, sm.cls, acc, my_node, nullptr, &pk);
            if (AFF && pk && S.cf.predicates) pk = aff_pred(S.aff, sm.cls_aff, S.N, my_node);     // list entries from L2: once per task
          }
          if (S.cf.fit_mode != 2 && (sm.pred_any_all || __any_sync(FULL, pk))) {      // fit_mode 2: a node that passes the predicates is IN the list
            if (lane == 0) {
              kb_decision d;
              d.node = -1; d.kind = KB_KIND_ALLOCATED; d.dispatched = 0; d.reserved = 0;
              d.step = 0xFFFFFFFFu; d.dispatch_step = 0xFFFFFFFFu;
              S.dec[task] = d;
            }
            n_phantom += 1;
          }
        }
        reason = STOP_NOFIT; break;
      }
      const uint32_t owner = (uint32_t)__ffs(__ballot_sync(FULL, cur_key == best)) - 1u;
      const unsigned ownbits = __shfl_sync(FULL, (next_valid ? 1u : 0u) | (cur_fi ? 2u : 0u), owner);
      if (BF && S.cf.fit_mode == 2 && !(ownbits & 2u)) {
        // backfill with the predicates plugin (EvalConf.fit_mode 2): the FIRST node that passes ssn.PredicateFn is tried and
        // node.AddTask refuses it (Resreq > Idle): ssn.Allocate has already made the task Allocated (session.go:241-262), it
        // has no node, and from now on InterPodAffinityMatches returns an error for every pair of the session (Ctl.pred_dead)
        if (lane == 0) {
          kb_decision d;
          d.node = -1; d.kind = KB_KIND_ALLOCATED; d.dispatched = 0; d.reserved = 0;
          d.step = 0xFFFFFFFFu; d.dispatch_step = 0xFFFFFFFFu;
          S.dec[task] = d;
          c.pred_dead = 1;
        }
        n_phantom += 1;
        cur_key = 0; next_key = 0; next_valid = true;
        reason = STOP_NOFIT; break;
      }
      if (!(ownbits & 1u)) refresh();
      const bool fits_idle = (ownbits & 2u) != 0;
      // commit: ssn.Allocate (session.go:235) or ssn.Pipeline (session.go:194) -> NodeInfo.AddTask (node_info.go:172-212):
      // the owner lane switches to its pre-evaluated next state
      if ((uint32_t)lane == owner) {
        my_cnt += 1;
        which ^= 1u;
        cur_key = next_key; cur_fi = next_fi; next_valid = false; modified = true;
      }
      // AllocateFunc handlers of drf (drf.go:136-144) and proportion (proportion.go:213-222)
      jalloc = KB_DADD(jalloc, my_rq);
      qalloc = KB_DADD(qalloc, my_rq);
      if (lane == 0) {
        kb_decision d;
        d.node = (int32_t)key_node(best);
        d.kind = fits_idle ? KB_KIND_ALLOCATED : KB_KIND_PIPELINED;
        d.dispatched = 0; d.reserved = 0;
        d.step = step0 + placed;
        d.dispatch_step = 0xFFFFFFFFu;
        S.dec[task] = d;
        if (AFF) aff_commit(S.aff, sm.cls_aff, S.N, key_node(best), fits_idle);
      }
      if (AFF) aff_stop = aff_rd;
      placed += 1;
      n_alloc += fits_idle ? 1u : 0u;
      // allocate.go:185-188: a ready job yields after every task while tasks remain
      const bool jr = !S.gang_ready || (ready + (int32_t)n_alloc) >= min_avail;     // ssn.JobReady
      if (!BF && jr && (pos + 1 < jend)) { reason = STOP_YIELD; break; }
      if (AFF && aff_stop) { if (run_left > 0) reason = STOP_RESCAN; break; }
    }
    // write the job-level state back, then run the control plane
    if (lane == 0) {
      S.job_pos[j] = pos0 + popped;
      S.job_ready[j] = ready + (int32_t)n_alloc + (int32_t)n_phantom;
      S.job_placed[j] += placed;
      c.step = step0 + placed;
      c.tasks_processed += popped;
      c.pairs_logical += (unsigned long long)popped * S.N;
      c.tasks_allocated += n_alloc;
      c.tasks_pipelined += placed - n_alloc;
      c.phantoms += n_phantom;
    }
    if (lane < R && placed) {
      if (S.drf_present) S.job_alloc[(size_t)lane * S.J + j] = jalloc;
      if (S.proportion_present) S.q_allocated[(size_t)lane * S.Q + q] = qalloc;
    }
    // drf.calculateShare (drf.go:161-171) / proportion.updateShare (proportion.go:241-253): one FP64 division per
    // dimension, all dimensions at once in lanes 0..R-1, then a max over the lanes (shares are >= 0, so the IEEE bit
    // patterns order like the values)
    if (placed) {
      if (S.drf_present) {
        double v = 0.0;
        if ((uint32_t)lane < R && ((S.total_dims_mask >> lane) & 1u)) v = share_of(jalloc, total_of<CR::CAP>(S, lane));
        const uint64_t m = warp_max_u64(double_as_u64(v));
        if (lane == 0) S.job_share[j] = u64_as_double(m);
      }
      if (S.proportion_present) {
        double v = 0.0;
        const uint32_t present = S.q_deserved_present[q] | 3u;
        if ((uint32_t)lane < R && ((present >> lane) & 1u)) v = share_of(qalloc, S.q_deserved[(size_t)lane * S.Q + q]);
        const uint64_t m = warp_max_u64(double_as_u64(v));
        if (lane == 0) S.q_share[q] = u64_as_double(m);
      }
    }
    __syncwarp();
    const long long t_run1 = clock64();
    if (lane == 0) {
      if (reason == STOP_RESCAN) c.rescans += 1;
      after_run<BF, CR::CAP>(S, c, reason, placed, true);
      const long long t_run2 = clock64();
      c.cyc_steps += (unsigned long long)(t_run1 - t_run0);
      c.cyc_ctl += (unsigned long long)(t_run2 - t_run1);
    }
    __syncwarp();
    if (reason == STOP_RESCAN) { rescanned = true; break; }
  }

  // write the modified candidates back to the global table
  if (modified) {
    const uint64_t (*src)[32] = sm.slot[which];
    for (uint32_t cc = 0; cc < ncols; ++cc) gt_mine[(size_t)cc * TILE_NODES] = src[cc][lane];
    for (uint32_t k = 0; k < R; ++k) {             // Used.Add(Resreq) once per placement (node_info.go:203)
      double u = S.node_used[(size_t)k * S.N + my_node];     // L1 hit: prefetched by the shadow warp
      for (uint32_t i = 0; i < my_cnt; ++i) u = KB_DADD(u, sm.cls.resreq[k]);
      S.node_used[(size_t)k * S.N + my_node] = u;
    }
  }
  __syncwarp();
  if (CH) {
    // what a following patch needs: this replay's modified candidates keep their CURRENT record in sm.slot[which]
    sm.lane_node[lane] = my_node; sm.lane_which[lane] = which; sm.lane_mod[lane] = modified ? 1u : 0u;
    bool add = modified;
    const uint32_t nm = sm.nmod;
    if (add) for (uint32_t i = 0; i < nm; ++i) if (sm.mod[i] == my_node) { add = false; break; }
    const unsigned mm = __ballot_sync(FULL, add);
    if (add) sm.mod[nm + __popc(mm & ((1u << lane) - 1u))] = my_node;
    if (lane == 0) { sm.nmod_prev = nm; sm.nmod = nm + __popc(mm); sm.last_rescan = rescanned ? 1u : 0u; }
    __threadfence();                          // the write-backs are visible before the next gather / patch re-reads records
    __syncwarp();
  }
  if (patch_class != 0xFFFFFFFFu) {
    // overlap mode: fresh keys of MY candidate (the scanners skipped it) for the class they scanned meanwhile
    const bool hit = !c.done && c.cur_class == patch_class;
    if (hit) {
      {
        const uint32_t* src = reinterpret_cast<const uint32_t*>(&class_table<CR>(S)[patch_class]);
        uint32_t* dst = reinterpret_cast<uint32_t*>(&sm.cls);
        for (uint32_t i = lane; i < sizeof(CR) / 4; i += 32) dst[i] = src[i];
      }
      __syncwarp();
      uint64_t pk = 0;
      if (have) {
        ColAcc acc{&sm.slot[which][0][0], (uint32_t)lane, 32u, R, W};
        pk = eval_pair(S.cf, sm.cls, acc, my_node, nullptr);
      }
      const unsigned n = __popc(__ballot_sync(FULL, have));
      pk = warp_sort_desc(pk, lane);
      c.patch[lane] = pk;
      if (lane == 0) { c.patch_valid = 1; c.pairs_replayed += (unsigned long long)n; }
    } else if (lane == 0) c.patch_valid = 0;
  }
  __syncwarp();
  if (lane == 0) {
    const long long t_end = clock64();
    c.cyc_scan += (unsigned long long)(t_scan - t_start);
    c.cyc_merge += (unsigned long long)(t_merge - t_scan);
    c.cyc_replay += (unsigned long long)(t_end - t_merge);
    if (patch_class == 0xFFFFFFFFu) c.cyc_total += (unsigned long long)(t_end - t_start);
  }
  __syncwarp();
}

// ---------------------------------------------------------------------------------------------
// Scan phase of one scanner CTA: tile GROUPS scanner_idx, +n_scanners, ... (S.tpi tiles per iteration, double-buffered
// TMA), K1+K2 per node against sm.cls, warp-level top-32, CTA tree fold.  Nodes listed in sm.excl (overlap mode) are
// skipped.  Every thread of the CTA calls it; the CTA's list is returned in warp 0.
// ---------------------------------------------------------------------------------------------
// thread 0 of a scanner CTA: start the bulk copies of its first tile group into staging buffer 0 (returns whether the
// CTA has any group).  The tiles do not depend on the class, so visit_kernel issues this BEFORE it reads the control
// block; scan_phase is then told that buffer 0 is already in flight.
template <class CR>
__device__ __forceinline__ bool issue_first_group(const DevSession& S, VisitSmem<CR>& sm, uint64_t* tilebuf, const uint32_t scanner_idx) {
  const uint32_t tile_u64 = S.ncols * TILE_NODES;
  const uint32_t tile_bytes = tile_u64 * 8u;
  const uint32_t tpi = S.tpi;
  const uint32_t n_groups = (S.tile_hi - S.tile_lo + tpi - 1) / tpi;
  if (scanner_idx >= n_groups) return false;
  const uint32_t t0 = S.tile_lo + scanner_idx * tpi;
  const uint32_t cnt = min(tpi, S.tile_hi - t0);
  mbar_expect_tx(&sm.mbar[0], cnt * tile_bytes);
  for (uint32_t k = 0; k < cnt; ++k)
    tma_load_1d(tilebuf + (size_t)k * tile_u64, S.tiles + (size_t)(t0 + k) * tile_u64, tile_bytes, &sm.mbar[0]);
  return true;
}

template <bool PH = false, int AFF = 0, class CR>
__device__ __forceinline__ uint64_t scan_phase(const DevSession& S, VisitSmem<CR>& sm, uint64_t* tilebuf, const uint32_t scanner_idx,
                                               const uint32_t n_scanners, const uint32_t cls_id, const int tid, const int lane, const int warp,
                                               const bool first_issued = false, const bool pred_dead = false) {
  const uint32_t tile_u64 = S.ncols * TILE_NODES;
  const uint32_t tile_bytes = tile_u64 * 8u;
  // ---------------- scan: tile GROUPS blockIdx.x, +gridDim.x, ...: S.tpi tiles per iteration, double-buffered TMA ----------------
  const uint32_t tpi = S.tpi;                                        // tiles per iteration (<= MAX_TPI, sized to shared memory)
  const uint32_t n_groups = (S.tile_hi - S.tile_lo + tpi - 1) / tpi;
  const uint32_t firstg = scanner_idx, stride = n_scanners;
  const uint32_t n_local = firstg < n_groups ? (n_groups - firstg + stride - 1) / stride : 0;
  auto issue_group = [&](uint32_t grp, uint32_t buf) {                 // thread 0: one bulk copy per tile of the group
    const uint32_t t0 = S.tile_lo + grp * tpi;
    const uint32_t cnt = min(tpi, S.tile_hi - t0);
    mbar_expect_tx(&sm.mbar[buf], cnt * tile_bytes);
    for (uint32_t k = 0; k < cnt; ++k)
      tma_load_1d(tilebuf + ((size_t)buf * tpi + k) * tile_u64, S.tiles + (size_t)(t0 + k) * tile_u64, tile_bytes, &sm.mbar[buf]);
  };
  if (tid == 0 && n_local > 0 && !first_issued) issue_group(firstg, 0);
  {
    // class record -> shared memory (broadcast reads afterwards) while the first tiles are in flight
    const uint32_t* src = reinterpret_cast<const uint32_t*>(&class_table<CR>(S)[cls_id]);
    uint32_t* dst = reinterpret_cast<uint32_t*>(&sm.cls);
    for (uint32_t i = tid; i < sizeof(CR) / 4; i += SCAN_THREADS) dst[i] = src[i];
    if (AFF) {
      const uint32_t* as = reinterpret_cast<const uint32_t*>(&S.aff.cls[cls_id]);
      uint32_t* ad = reinterpret_cast<uint32_t*>(&sm.cls_aff);
      for (uint32_t i = tid; i < sizeof(ClassAff) / 4; i += SCAN_THREADS) ad[i] = as[i];
      if (S.aff.has_x) {
        const uint32_t xn = min(S.aff.cls[cls_id].xf_cnt, AFF_XF_SMEM), xo = S.aff.cls[cls_id].xf_off;
        for (uint32_t i = tid; i < xn; i += SCAN_THREADS) sm.cls_xf[i] = S.aff.xf[xo + i];
      }
      uint32_t* pd = reinterpret_cast<uint32_t*>(&sm.cls_pref);
      if (S.aff.has_pref) {
        const uint32_t* ps = reinterpret_cast<const uint32_t*>(&pref_table<CR>(S)[cls_id]);
        for (uint32_t i = tid; i < sizeof(ClassPrefOf<CR>) / 4; i += SCAN_THREADS) pd[i] = ps[i];
      } else if (tid == 0) sm.cls_pref.n = 0;
    }
  }
  __syncthreads();
  // InterPodAffinityPriority: the passes of aff_prepass_kernel left the per-domain weights and the min / max count
  const bool ipa = AFF && sm.cls_aff.w_cnt != 0 && S.cf.nodeorder != 0;
  const long long ipa_min = ipa ? __ldcg(&S.aff.minmax[0]) : 0ll, ipa_max = ipa ? __ldcg(&S.aff.minmax[1]) : 0ll;
  // NodeAffinityPriority on the per-visit kernels: pass 2 left the max count over the feasible nodes (NormalizeReduce, reduce.go:28-63)
  const bool prf = AFF && S.aff.has_pref && sm.cls_pref.n != 0 && S.cf.nodeorder != 0;
  const long long prf_max = prf ? __ldcg(&S.aff.minmax[2]) : 0ll;
  const uint32_t sub = (uint32_t)warp >> 2, part = (uint32_t)warp & 3u;    // which tile of the group / which 32 nodes of it
  uint64_t mylist = 0;                       // this warp's running top-32 (lane l holds the l-th best)
  bool pany = false;                         // PH (backfill): a node that passes the plugin predicates but has no Idle for Resreq
  for (uint32_t it = 0; it < n_local; ++it) {
    const uint32_t b = it & 1u;
    if (it + 1 < n_local) {
      __syncthreads();                       // every thread is done reading the other buffer (iteration it-1)
      if (tid == 0) issue_group(firstg + (it + 1) * stride, b ^ 1u);
    }
    mbar_wait(&sm.mbar[b], (it >> 1) & 1u);
    const uint32_t t = S.tile_lo + (firstg + it * stride) * tpi + sub;
    const uint32_t node = t * TILE_NODES + part * 32u + lane;
    uint64_t key = 0;
    // overlap mode: the replayer CTA may be modifying these nodes right now; it contributes their keys itself
    unsigned exmask = 0;
    if (sm.n_excl) {
      const uint32_t d = sm.excl[lane] - (t * TILE_NODES + part * 32u);
      exmask = __reduce_or_sync(FULL, ((uint32_t)lane < sm.n_excl && d < 32u) ? (1u << d) : 0u);
    }
    if (sub < tpi && t < S.tile_hi && node < S.N && !((exmask >> lane) & 1u)) {
      ColAcc acc{tilebuf + ((size_t)b * tpi + sub) * tile_u64, part * 32u + lane, TILE_NODES, S.cf.R, S.cf.W};
      bool pok = false;
      key = eval_pair(S.cf, sm.cls, acc, node, nullptr, PH ? &pok : nullptr);
      if (PH && pred_dead) { key = 0; pok = false; }        // a task Allocated on no node: InterPodAffinityMatches errors for every pair (Ctl.pred_dead)
      if (AFF) {
        if (S.cf.predicates && !aff_pred(S.aff, sm.cls_aff, S.N, node, sm.cls_xf, AFF_XF_SMEM)) { key = 0; pok = false; }   // predicate step 10
        if (ipa && key) key = aff_add_score(key, S.aff.w_podaff, aff_score(aff_count_node(S.aff, sm.cls_aff, S.N, node), ipa_min, ipa_max));
        if (prf && key) key = add_pref_term(key, (int64_t)S.w_nodeaff, (int64_t)pref_count(sm.cls_pref, acc, S.cf.W), (int64_t)prf_max);
      }
      if (PH) pany = pany | (pok && key == 0);
    }
    // K3, warp level: skip the networks when nothing in this warp can enter its list
    const uint64_t thr = __shfl_sync(FULL, mylist, 31);
    if (__any_sync(FULL, key > thr)) {
      key = warp_sort_desc(key, lane);
      mylist = warp_merge_top32(mylist, key, lane);
    }
  }
  if (PH) { if (__any_sync(FULL, pany) && lane == 0) atomicOr(&sm.pred_any, 1u); }
  // CTA level: tree-fold the warps' lists into warp 0, which publishes the CTA's list
  mylist = cta_fold_lists(mylist, sm.wlist, warp, lane);
  return mylist;
}

__device__ __forceinline__ void load_ctl(Ctl& dst, const Ctl* g, int lane) {
  const uint32_t* src = reinterpret_cast<const uint32_t*>(g);
  uint32_t* d = reinterpret_cast<uint32_t*>(&dst);
  for (uint32_t i = lane; i < sizeof(Ctl) / 4; i += 32) d[i] = __ldcg(src + i);
}

// Several queues: the Go-heap emulation's next pop sifts down from the root and its next push climbs from the tail.  Pull the
// top 12 levels of qheap (one load per line), the tail's ancestors, and the rows of the queues the first comparisons read: the
// top 5 levels (31 entries) and the tail's ancestor chain — share, ctime, job-list cursors, deserved / allocated and, with HEAD,
// the head job of their static lists — plus the re-pushed jobs of the root's queue.  At most three queue rows per lane per call,
// whatever Q is.
template <bool HEAD>
__device__ __forceinline__ uint32_t prefetch_queue_heap(const DevSession& S, const uint32_t len, const int lane) {
  const uint32_t R = S.cf.R;
  uint32_t acc = 0;
  for (uint32_t i = (uint32_t)lane * 32u; i < len && i < 4096u; i += 1024u) acc += S.qheap[i];
  auto row = [&](const uint32_t qq) {
    acc += (uint32_t)double_as_u64(S.q_share[qq]) + (uint32_t)S.q_ctime[qq] + S.q_static_head[qq] + S.q_static_off[qq + 1] + S.q_dyn_len[qq];
    for (uint32_t k = 0; k < R; ++k)
      acc += (uint32_t)double_as_u64(S.q_deserved[(size_t)k * S.Q + qq]) + (uint32_t)double_as_u64(S.q_allocated[(size_t)k * S.Q + qq]);
    if (HEAD) {
      const uint32_t hq = S.q_static_head[qq];
      if (hq < S.q_static_off[qq + 1]) {
        const uint32_t jn = S.q_static[hq];
        const uint32_t pn = S.job_pos[jn];
        acc += (uint32_t)S.job_ready[jn] + (uint32_t)S.job_min_avail[jn] + S.job_ord_off[jn + 1] + S.ord_class[pn] + S.ord_run[pn] + S.ord_task[pn];
      }
    }
  };
  if (lane < 31 && (uint32_t)lane < len) row(S.qheap[lane]);
  const uint32_t up = ((len + 1) >> lane);                 // ancestors of the push position `len`
  if (up >= 1 && up - 1 < len) row(S.qheap[up - 1]);
  if (len) row(S.qheap[len - 1]);                          // moves to the root on the next pop
  if (len) {
    const uint32_t q0 = S.qheap[0];
    if ((uint32_t)lane < S.q_dyn_len[q0]) acc += S.dyn_jobs[S.q_static_off[q0] + lane];
  }
  return acc;
}

// ---------------------------------------------------------------------------------------------
// Shadow prefetch (warp 1 of the last CTA, concurrent with warp 0's gather / look-ahead / steps): touch the
// job-level state of the current visit and what select_next_visit / setup_run will most likely read next (the head of
// the queue's static job list), so that warp 0 finds it in L1 instead of paying a chain of L2 round trips.
// Read-only; the sum goes to `sink` only to keep the loads alive.
// ---------------------------------------------------------------------------------------------
template <int BF>
__device__ __forceinline__ void shadow_prefetch(const DevSession& S, const Ctl& c, const int lane, uint32_t* sink, const uint64_t cand_key) {
  if (BF || c.done || c.cur_job < 0) return;
  const uint32_t j = (uint32_t)c.cur_job, q = c.cur_queue, R = S.cf.R;
  uint32_t acc = 0;
  if (cand_key)                                   // NodeInfo.Used rows of this lane's candidate (read at write-back time)
    for (uint32_t k = 0; k < R; ++k) acc += (uint32_t)double_as_u64(S.node_used[(size_t)k * S.N + key_node(cand_key)]);
  const uint32_t pos = S.job_pos[j], end = S.job_ord_off[j + 1];
  acc += (uint32_t)S.job_ready[j] + (uint32_t)S.job_min_avail[j] + S.job_placed[j];
  if (pos + lane < end) acc += S.ord_task[pos + lane];
  if ((uint32_t)lane < R) {
    acc += (uint32_t)double_as_u64(S.job_alloc[(size_t)lane * S.J + j]);
    acc += (uint32_t)double_as_u64(S.q_allocated[(size_t)lane * S.Q + q]) + (uint32_t)double_as_u64(S.q_deserved[(size_t)lane * S.Q + q]);
  }
  acc += S.q_deserved_present[q] + (uint32_t)double_as_u64(S.q_share[q]) + (uint32_t)double_as_u64(S.job_share[j]);
  const uint32_t h = S.q_static_head[q];
  if (h < S.q_static_off[q + 1]) {
    const uint32_t jn = S.q_static[h];
    const uint32_t pn = S.job_pos[jn], en = S.job_ord_off[jn + 1];
    acc += (uint32_t)S.job_ready[jn] + (uint32_t)S.job_min_avail[jn] + S.job_placed[jn] + S.job_queue[jn];
    if (pn < en) acc += S.ord_class[pn] + S.ord_run[pn];
    if (pn + lane < en) acc += S.ord_task[pn + lane];
    if ((uint32_t)lane < R) acc += (uint32_t)double_as_u64(S.job_alloc[(size_t)lane * S.J + jn]);
  }
  if (S.Q > 1) acc += prefetch_queue_heap<false>(S, c.qheap_len, lane);
  acc = __reduce_add_sync(FULL, acc);
  if (lane == 0) *sink = acc;
}

// ---------------------------------------------------------------------------------------------
// visit_kernel
// ---------------------------------------------------------------------------------------------
// CR: class record type of the session (ClassRecNarrow, ClassRecWide for R > KB_NARROW_R, ClassRecAtoms for W > KB_NARROW_W): the
// class record, its preferred terms and the candidate slots
template <int BF, int AFF = 0, class CR = ClassRecNarrow>
__global__ void __launch_bounds__(SCAN_THREADS)
visit_kernel(const __grid_constant__ DevSession S) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  // layout: [VisitSmem][pad to 128][tile buffer 0][tile buffer 1]
  VisitSmem<CR>& sm = *reinterpret_cast<VisitSmem<CR>*>(smem_raw);
  uint64_t* tilebuf = reinterpret_cast<uint64_t*>(smem_raw + ((sizeof(VisitSmem<CR>) + 127) / 128) * 128);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  Ctl* gctl = S.ctl;
  if (tid == 0) { mbar_init(&sm.mbar[0], 1); mbar_init(&sm.mbar[1], 1); fence_mbar_init(); sm.n_excl = 0; sm.pred_any = 0; sm.pred_any_all = 0; }
  if (tid < 32) sm.excl[tid] = 0;
  // programmatic dependent launch: this grid may have been scheduled while the previous launch was still replaying;
  // nothing the previous launch writes is read before this point (no-op when launched without the attribute)
  pdl_wait();
  // the node tiles do not depend on the class: start staging them before the control block is even read
  bool in_flight = false;
  if (tid == 0) in_flight = issue_first_group(S, sm, tilebuf, blockIdx.x);
  if (*((volatile uint32_t*)&gctl->done)) {
    if (in_flight) mbar_wait(&sm.mbar[0], 0);        // a CTA must not exit with bulk copies into its shared memory in flight
    return;
  }
  const uint32_t cls_id = *((volatile uint32_t*)&gctl->cur_class);
  __syncthreads();
  const long long t_start = clock64();

  const bool pred_dead = BF && *((volatile uint32_t*)&gctl->pred_dead) != 0;
  uint64_t mylist = scan_phase<BF != 0, AFF>(S, sm, tilebuf, blockIdx.x, gridDim.x, cls_id, tid, lane, warp, true, pred_dead);
  if (warp == 0) {
    S.cand[(size_t)blockIdx.x * KTOP + lane] = mylist;
    if (BF && lane == 0) S.cand[((size_t)gridDim.x + blockIdx.x) * KTOP] = (uint64_t)sm.pred_any;      // second bank of the list area
    sm.keys[lane] = mylist;
    __threadfence();
    __syncwarp();                            // every lane's list entry is fenced before the ticket is taken
    if (lane == 0) {
      const uint32_t ticket = atomicAdd(&gctl->arrive, 1u);
      sm.is_last = (ticket == gridDim.x - 1) ? 1u : 0u;
    }
  }
  __syncthreads();
  if (!sm.is_last) return;
  __threadfence();
  pdl_launch_dependents();                   // every other CTA has exited: the next launch can be scheduled while this CTA replays
  const long long t_scan = clock64();
  // control block: the loads are issued now by the last warp and land in registers while everybody merges
  constexpr int CTLW = (int)((sizeof(Ctl) / 4 + 31) / 32);
  uint32_t cw[CTLW];
  if (warp == SCAN_WARPS - 1) {
#pragma unroll
    for (int i = 0; i < CTLW; ++i) {
      const uint32_t idx = (uint32_t)i * 32u + lane;
      cw[i] = idx < sizeof(Ctl) / 4 ? __ldcg(reinterpret_cast<const uint32_t*>(gctl) + idx) : 0u;
    }
  }

  if (BF && warp == 1) {                     // backfill: OR of the CTAs' "a node outside the lists passes the predicates" bits
    uint32_t f = 0;
    for (uint32_t g2 = lane; g2 < gridDim.x; g2 += 32) f |= (uint32_t)__ldcg(&S.cand[((size_t)gridDim.x + g2) * KTOP]);
    f = __reduce_or_sync(FULL, f);
    if (lane == 0) sm.pred_any_all = f;
  }
  // ---------------- K3: merge the per-CTA lists: every warp folds every 16th list, then the tree ----------------
  if (gridDim.x > 1) {
    const uint32_t G = gridDim.x;
    uint64_t acc = 0;
    uint32_t g = warp;
    uint64_t nxt = g < G ? __ldcg(&S.cand[(size_t)g * KTOP + lane]) : 0ull;
    while (g < G) {
      const uint64_t cur = nxt;
      const uint32_t g2 = g + SCAN_WARPS;
      nxt = g2 < G ? __ldcg(&S.cand[(size_t)g2 * KTOP + lane]) : 0ull;     // prefetch the next list
      const uint64_t thr = __shfl_sync(FULL, acc, 31);
      const uint64_t head = __shfl_sync(FULL, cur, 0);
      if (head > thr) acc = warp_merge_top32(acc, cur, lane);
      g = g2;
    }
    acc = cta_fold_lists(acc, sm.wlist, warp, lane);
    if (warp == 0) sm.keys[lane] = acc;
  }
  if (S.world > 1 && S.p2p) {
    // ---------------- fused exchange over peer memory (NVLink): no NCCL, no second kernel ----------------
    // Every rank pushes its top-32 keys + the candidates' node records into each peer's recv slot [parity][rank],
    // fences system-wide, raises its flag there, then waits for all peers' flags in its own region.  A rank can run at
    // most one scan ahead of a peer (it needs the peer's block to finish), so two parities are enough.
    __syncthreads();
    const uint32_t epoch = *((volatile uint32_t*)&gctl->xchg_epoch);
    const uint32_t par = epoch & 1u;
    if (warp == 0) {
      const uint64_t k = sm.keys[lane];
      if (k) {
        const uint32_t n = key_node(k);
        const uint64_t* rec = S.tiles + (size_t)(n / TILE_NODES) * ((size_t)S.ncols * TILE_NODES) + (n % TILE_NODES);
        for (uint32_t cc = 0; cc < S.ncols; ++cc) sm.slot[0][cc][lane] = __ldcg(rec + (size_t)cc * TILE_NODES);
      }
    }
    __syncthreads();
    if ((uint32_t)warp < S.world) {
      uint64_t* dst = S.peer_base[warp] + (size_t)(par * KB_MAX_WORLD + S.rank) * P2P_RANK_U64;
      dst[lane] = sm.keys[lane];
      for (uint32_t cc = 0; cc < S.ncols; ++cc) dst[(size_t)(1 + cc) * 32 + lane] = sm.slot[0][cc][lane];
      if (BF) dst[(size_t)(1 + S.ncols) * 32 + lane] = (uint64_t)sm.pred_any_all;
      __threadfence_system();
      __syncwarp();
      if (lane == 0) *((volatile uint64_t*)(S.peer_base[warp] + P2P_FLAG_OFF + par * KB_MAX_WORLD + S.rank)) = (uint64_t)epoch;
    }
    if (warp == 1) { load_ctl(sm.ctl2, gctl, lane); __syncwarp(); shadow_prefetch<BF>(S, sm.ctl2, lane, &sm.sink, 0ull); }
    if (warp != 0) return;
    // wait for every rank's block (bounded: ~2 s at 2 GHz, then the cycle is aborted with an error)
    {
      const volatile uint64_t* fl = S.peer_base[S.rank] + P2P_FLAG_OFF + par * KB_MAX_WORLD + lane;
      const long long deadline = clock64() + 4000000000ll;
      bool ok = true;
      while ((uint32_t)lane < S.world && *fl != (uint64_t)epoch) {
        if (clock64() > deadline) { ok = false; break; }
      }
      if (!__all_sync(FULL, ok)) {
        if (lane == 0) { gctl->error = 2; gctl->done = 1; gctl->arrive = 0; }
        return;
      }
    }
    __threadfence();
    const uint64_t* recv = S.peer_base[S.rank] + (size_t)par * KB_MAX_WORLD * P2P_RANK_U64;
    uint64_t acc = __ldcg(recv + lane);
    for (uint32_t r = 1; r < S.world; ++r) acc = warp_merge_top32(acc, __ldcg(recv + (size_t)r * P2P_RANK_U64 + lane), lane);
    sm.keys[lane] = acc;
    if (BF) {
      uint32_t f = (uint32_t)lane < S.world ? (uint32_t)__ldcg(recv + (size_t)lane * P2P_RANK_U64 + (size_t)(1 + S.ncols) * 32) : 0u;
      f = __reduce_or_sync(FULL, f);
      if (lane == 0) sm.pred_any_all = f;
      __syncwarp();
    }
    const uint32_t node = key_node(acc);
    uint32_t owner = node / S.nodes_per_rank;
    owner = owner < S.world ? owner : S.world - 1;
    uint32_t idx = 0;
    if (acc)
      for (uint32_t i = 0; i < 32; ++i)
        if (__ldcg(recv + (size_t)owner * P2P_RANK_U64 + i) == acc) idx = i;
    load_ctl(sm.ctl, gctl, lane);
    __syncwarp();
    replay_epilogue<BF>(S, sm, lane, cls_id, recv + (size_t)owner * P2P_RANK_U64 + 32 + idx, 32u, 0xFFFFFFFFu, t_start, t_scan);
    if (lane == 0) sm.ctl.xchg_epoch = epoch + 1;
    __syncwarp();
    store_ctl(gctl, sm.ctl, lane);
    if (lane == 0) gctl->arrive = 0;
    return;
  }
  if (S.world > 1) {
    // sharded node axis: publish this rank's candidates WITH their node records; the replay happens in
    // replay_kernel after the all-gather
    __syncthreads();
    if (warp == 0) {
      const uint64_t k = sm.keys[lane];
      S.sendbuf[lane] = k;
      if (BF) S.sendbuf[(size_t)(1 + S.ncols) * 32 + lane] = (uint64_t)sm.pred_any_all;
      if (k) {
        const uint32_t n = key_node(k);
        const uint64_t* rec = S.tiles + (size_t)(n / TILE_NODES) * ((size_t)S.ncols * TILE_NODES) + (n % TILE_NODES);
        for (uint32_t cc = 0; cc < S.ncols; ++cc) S.sendbuf[(size_t)(1 + cc) * 32 + lane] = __ldcg(rec + (size_t)cc * TILE_NODES);
      }
    }
    return;
  }
  if (warp == SCAN_WARPS - 1) {
#pragma unroll
    for (int i = 0; i < CTLW; ++i) {
      const uint32_t idx = (uint32_t)i * 32u + lane;
      if (idx < sizeof(Ctl) / 4) reinterpret_cast<uint32_t*>(&sm.ctl)[idx] = cw[i];
    }
  }
  __syncthreads();
  if (warp == 1) shadow_prefetch<BF>(S, sm.ctl, lane, &sm.sink, sm.keys[lane]);
  if (warp != 0) return;

  // ---------------- exact replay + control: warp 0 only ----------------
  {
    const uint32_t n = key_node(sm.keys[lane]);
    const uint64_t* rec = S.tiles + (size_t)(n / TILE_NODES) * ((size_t)S.ncols * TILE_NODES) + (n % TILE_NODES);
    replay_epilogue<BF, 0, AFF>(S, sm, lane, cls_id, rec, TILE_NODES, 0xFFFFFFFFu, t_start, t_scan);
    store_ctl(gctl, sm.ctl, lane);
    if (lane == 0) gctl->arrive = 0;
  }
}

// ---------------------------------------------------------------------------------------------
// aff_prepass_kernel<PHASE>: InterPodAffinityPriority (vendor/.../priorities/interpod_affinity.go:99-235) needs two
// reductions over the FEASIBLE nodes before a single key of the visit's class exists; three small launches precede the
// visit_kernel of a session whose classes carry weight lists (they return at once for a class without one):
//   0  clear the per-domain weights and the min / max count
//   1  every feasible node adds the weight of its pods to the topology domain of the "pod's node" (kb_aff.h aff_pass1_node)
//   2  every feasible node's count = sum of its domains' weights -> min / max (both start at 0, :205-214)
// visit_kernel's scan then adds w * int(10 * (count - min) / (max - min)) to the key (pass 3).  Node records are read from the
// global tiles (L2 resident); feasible = K1 + predicate step 10, exactly the scan's test.
// ---------------------------------------------------------------------------------------------
constexpr int AFF_THREADS = 256;
template <int PHASE, class CR = ClassRecNarrow>
__global__ void __launch_bounds__(AFF_THREADS)
aff_prepass_kernel(const __grid_constant__ DevSession S) {
  __shared__ CR scls;
  __shared__ ClassAff sca;
  __shared__ AffX sxf[AFF_XF_SMEM];
  if (__ldcg(&S.ctl->done) || !S.cf.nodeorder) return;
  const uint32_t cls_id = __ldcg(&S.ctl->cur_class);
  const bool wts = S.aff.cls[cls_id].w_cnt != 0;
  const bool prf = S.aff.has_pref && pref_table<CR>(S)[cls_id].n != 0;        // NodeAffinityPriority: max count over the feasible nodes
  if (!wts && !prf) return;
  const uint32_t gtid = blockIdx.x * blockDim.x + threadIdx.x, nthr = gridDim.x * blockDim.x;
  if (PHASE == 0) {
    if (wts) for (uint32_t i = gtid; i < S.aff.dom_total; i += nthr) S.aff.dom_sum[i] = 0;
    if (gtid == 0) { S.aff.minmax[0] = 0; S.aff.minmax[1] = 0; S.aff.minmax[2] = 0; }
    return;
  }
  if (PHASE == 1 && !wts) return;
  __shared__ ClassPrefOf<CR> scp;
  if (prf) {
    const uint32_t* ps = reinterpret_cast<const uint32_t*>(&pref_table<CR>(S)[cls_id]);
    uint32_t* pd = reinterpret_cast<uint32_t*>(&scp);
    for (uint32_t i = threadIdx.x; i < sizeof(ClassPrefOf<CR>) / 4; i += blockDim.x) pd[i] = ps[i];
  }
  {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(&class_table<CR>(S)[cls_id]);
    uint32_t* dst = reinterpret_cast<uint32_t*>(&scls);
    for (uint32_t i = threadIdx.x; i < sizeof(CR) / 4; i += blockDim.x) dst[i] = src[i];
    const uint32_t* as = reinterpret_cast<const uint32_t*>(&S.aff.cls[cls_id]);
    uint32_t* ad = reinterpret_cast<uint32_t*>(&sca);
    for (uint32_t i = threadIdx.x; i < sizeof(ClassAff) / 4; i += blockDim.x) ad[i] = as[i];
    if (S.aff.has_x) {
      const uint32_t xn = min(S.aff.cls[cls_id].xf_cnt, AFF_XF_SMEM), xo = S.aff.cls[cls_id].xf_off;
      for (uint32_t i = threadIdx.x; i < xn; i += blockDim.x) sxf[i] = S.aff.xf[xo + i];
    }
  }
  __syncthreads();
  const size_t tile_u64 = (size_t)S.ncols * TILE_NODES;
  long long mn = 0, mx = 0;
  auto feasible = [&](const uint32_t n) {
    TileAcc acc{S.tiles + (size_t)(n / TILE_NODES) * tile_u64, n % TILE_NODES, S.cf.R, S.cf.W};
    uint64_t key = eval_pair(S.cf, scls, acc, n, nullptr);
    if (key && S.cf.predicates && !aff_pred(S.aff, sca, S.N, n, sxf, AFF_XF_SMEM)) key = 0;
    return key != 0;
  };
  if (PHASE == 1) {
    // one WARP per node: lane 0 decides feasibility, then the lanes share the class's weight list
    const uint32_t lane = threadIdx.x & 31u, gw = gtid >> 5, nw = nthr >> 5;
    for (uint32_t n = gw; n < S.N; n += nw) {
      const bool ok = __shfl_sync(0xFFFFFFFFu, (lane == 0 && feasible(n)) ? 1 : 0, 0) != 0;
      if (!ok) continue;
      aff_pass1_node(S.aff, sca, S.N, n, [&](uint32_t slot, long long v) {
        atomicAdd(reinterpret_cast<unsigned long long*>(&S.aff.dom_sum[slot]), (unsigned long long)v); }, lane, 32u);
    }
  } else {
    long long pmx = 0;
    for (uint32_t n = gtid; n < S.N; n += nthr) {
      if (!feasible(n)) continue;
      if (wts) {
        const long long cnt = aff_count_node(S.aff, sca, S.N, n);
        mn = cnt < mn ? cnt : mn; mx = cnt > mx ? cnt : mx;
      }
      if (prf) {
        TileAcc acc{S.tiles + (size_t)(n / TILE_NODES) * tile_u64, n % TILE_NODES, S.cf.R, S.cf.W};
        const long long pc = (long long)pref_count(scp, acc, S.cf.W);
        pmx = pc > pmx ? pc : pmx;
      }
    }
    if (pmx > 0) atomicMax(&S.aff.minmax[2], pmx);
  }
  if (PHASE == 2) {
    if (mn < 0) atomicMin(&S.aff.minmax[0], mn);
    if (mx > 0) atomicMax(&S.aff.minmax[1], mx);
  }
}

// ---------------------------------------------------------------------------------------------
// visit_chain_kernel<K> (single GPU): ONE pass over the node table serves up to K consecutive visits.
//   scan     every CTA evaluates cur_class AND the K-1 predicted classes of the following visits (Ctl.chain, from the
//            static job order) for each of its nodes: K exact top-32 lists per CTA, folded in log2(16) rounds that
//            spread the K x 16 warp lists over all warps;
//   merge    the last CTA folds the per-CTA lists of all classes at once (16/K warps per class);
//   replay   warp 0 replays the first visit as visit_kernel does.  While the control plane's next visit has the class
//            of an unused look-ahead list, that list is PATCHED — entries of nodes modified since the scan are dropped,
//            those nodes are re-evaluated from their current records, the 32 best stay and the certification floor rises
//            to the best key that did not fit — and replayed in the same launch.
// Exactness: an unmodified node outside a look-ahead list still has a key below that list's floor; every modified node
// is re-evaluated; keys are unique (node index), so "best >= floor" certifies a pick exactly as in visit_kernel.
// A wrong prediction only wastes the look-ahead evaluation.  tests/emu mirrors this protocol (emu_launch_chain).
// ---------------------------------------------------------------------------------------------
template <int K, class CR = ClassRecNarrow>
struct ChainSmem {
  CR cls[K];
  uint32_t cls_id[K];
  uint64_t keys[K][KTOP];                    // merged list per class (launch-start state)
  uint64_t fold[2][K][SCAN_WARPS][KTOP];     // ping-pong buffers of the fold rounds
};
template <int K, class CR = ClassRecNarrow>
__host__ __device__ constexpr size_t chain_smem_header() {
  return ((sizeof(VisitSmem<CR>) + 127) / 128) * 128 + ((sizeof(ChainSmem<K, CR>) + 127) / 128) * 128;
}

// one fold round over lists of `nK` classes: n lists per class in buf[cur] -> n/2 in buf[cur^1]; jobs spread over the warps
template <int K, class CR>
__device__ __forceinline__ void chain_fold_round(ChainSmem<K, CR>& cs, const int cur, const int n, const int nK, const int warp, const int lane) {
  const int half = n >> 1, jobs = nK * half;
  for (int t = warp; t < jobs; t += SCAN_WARPS) {
    const int k = t / half, i = t - k * half;
    cs.fold[cur ^ 1][k][i][lane] = warp_merge_top32(cs.fold[cur][k][2 * i][lane], cs.fold[cur][k][2 * i + 1][lane], lane);
  }
  __syncthreads();
}

template <int K, class CR = ClassRecNarrow>
__global__ void __launch_bounds__(SCAN_THREADS)
visit_chain_kernel(const __grid_constant__ DevSession S) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  VisitSmem<CR>& sm = *reinterpret_cast<VisitSmem<CR>*>(smem_raw);
  ChainSmem<K, CR>& cs = *reinterpret_cast<ChainSmem<K, CR>*>(smem_raw + ((sizeof(VisitSmem<CR>) + 127) / 128) * 128);
  uint64_t* tilebuf = reinterpret_cast<uint64_t*>(smem_raw + chain_smem_header<K, CR>());

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  Ctl* gctl = S.ctl;
  if (tid == 0) { mbar_init(&sm.mbar[0], 1); mbar_init(&sm.mbar[1], 1); fence_mbar_init(); sm.n_excl = 0; sm.nmod = 0; sm.nmod_prev = 0; sm.last_rescan = 0; sm.chain_seq = 0; }
  pdl_wait();
  if (*((volatile uint32_t*)&gctl->done)) return;
  if (tid < K) cs.cls_id[tid] = tid == 0 ? *((volatile uint32_t*)&gctl->cur_class) : *((volatile uint32_t*)&gctl->chain[tid - 1]);
  __syncthreads();
  int nK = 1;
  while (nK < K && cs.cls_id[nK] != 0xFFFFFFFFu) ++nK;
  const long long t_start = clock64();

  // ---------------- scan: as scan_phase, K classes per node ----------------
  const uint32_t tile_u64 = S.ncols * TILE_NODES;
  const uint32_t tile_bytes = tile_u64 * 8u;
  const uint32_t tpi = S.tpi;
  const uint32_t n_groups = (S.tile_hi - S.tile_lo + tpi - 1) / tpi;
  const uint32_t firstg = blockIdx.x, stride = gridDim.x;
  const uint32_t n_local = firstg < n_groups ? (n_groups - firstg + stride - 1) / stride : 0;
  auto issue_group = [&](uint32_t grp, uint32_t buf) {
    const uint32_t t0 = S.tile_lo + grp * tpi;
    const uint32_t cnt = min(tpi, S.tile_hi - t0);
    mbar_expect_tx(&sm.mbar[buf], cnt * tile_bytes);
    for (uint32_t k = 0; k < cnt; ++k)
      tma_load_1d(tilebuf + ((size_t)buf * tpi + k) * tile_u64, S.tiles + (size_t)(t0 + k) * tile_u64, tile_bytes, &sm.mbar[buf]);
  };
  if (tid == 0 && n_local > 0) issue_group(firstg, 0);
  for (int k = 0; k < nK; ++k) {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(&class_table<CR>(S)[cs.cls_id[k]]);
    uint32_t* dst = reinterpret_cast<uint32_t*>(&cs.cls[k]);
    for (uint32_t i = tid; i < sizeof(CR) / 4; i += SCAN_THREADS) dst[i] = src[i];
  }
  __syncthreads();
  const uint32_t sub = (uint32_t)warp >> 2, part = (uint32_t)warp & 3u;
  uint64_t mylist[K];
#pragma unroll
  for (int k = 0; k < K; ++k) mylist[k] = 0;
  for (uint32_t it = 0; it < n_local; ++it) {
    const uint32_t b = it & 1u;
    if (it + 1 < n_local) {
      __syncthreads();
      if (tid == 0) issue_group(firstg + (it + 1) * stride, b ^ 1u);
    }
    mbar_wait(&sm.mbar[b], (it >> 1) & 1u);
    const uint32_t t = S.tile_lo + (firstg + it * stride) * tpi + sub;
    const uint32_t node = t * TILE_NODES + part * 32u + lane;
    const bool valid = sub < tpi && t < S.tile_hi && node < S.N;
    ColAcc acc{tilebuf + ((size_t)b * tpi + sub) * tile_u64, part * 32u + lane, TILE_NODES, S.cf.R, S.cf.W};
#pragma unroll
    for (int k = 0; k < K; ++k) {
      if (k < nK) {
        uint64_t key = valid ? eval_pair(S.cf, cs.cls[k], acc, node, nullptr) : 0ull;
        const uint64_t thr = __shfl_sync(FULL, mylist[k], 31);
        if (__any_sync(FULL, key > thr)) {
          key = warp_sort_desc(key, lane);
          mylist[k] = warp_merge_top32(mylist[k], key, lane);
        }
      }
    }
  }
  // CTA fold: K x 16 warp lists -> K lists, 4 rounds
#pragma unroll
  for (int k = 0; k < K; ++k) if (k < nK) cs.fold[0][k][warp][lane] = mylist[k];
  __syncthreads();
  int cur = 0;
  for (int n = SCAN_WARPS; n > 1; n >>= 1) { chain_fold_round<K, CR>(cs, cur, n, nK, warp, lane); cur ^= 1; }
  const uint32_t G = gridDim.x;
  if (warp < nK) {
    const uint64_t v = cs.fold[cur][warp][0][lane];
    S.cand[((size_t)warp * G + blockIdx.x) * KTOP + lane] = v;
    cs.keys[warp][lane] = v;
    __threadfence();
  }
  __syncthreads();
  if (tid == 0) {
    const uint32_t ticket = atomicAdd(&gctl->arrive, 1u);
    sm.is_last = (ticket == G - 1) ? 1u : 0u;
  }
  __syncthreads();
  if (!sm.is_last) return;
  __threadfence();
  pdl_launch_dependents();
  const long long t_scan = clock64();
  constexpr int CTLW = (int)((sizeof(Ctl) / 4 + 31) / 32);
  uint32_t cw[CTLW];
  if (warp == SCAN_WARPS - 1) {
#pragma unroll
    for (int i = 0; i < CTLW; ++i) {
      const uint32_t idx = (uint32_t)i * 32u + lane;
      cw[i] = idx < sizeof(Ctl) / 4 ? __ldcg(reinterpret_cast<const uint32_t*>(gctl) + idx) : 0u;
    }
  }
  // ---------------- merge the per-CTA lists: 16/K warps per class, then log2(16/K) rounds ----------------
  if (G > 1) {
    constexpr int P = SCAN_WARPS / K;
    const int k = warp % K, p = warp / K;
    uint64_t acc = 0;
    if (k < nK) {
      uint32_t g = (uint32_t)p;
      uint64_t nxt = g < G ? __ldcg(&S.cand[((size_t)k * G + g) * KTOP + lane]) : 0ull;
      while (g < G) {
        const uint64_t c0 = nxt;
        const uint32_t g2 = g + P;
        nxt = g2 < G ? __ldcg(&S.cand[((size_t)k * G + g2) * KTOP + lane]) : 0ull;
        const uint64_t thr = __shfl_sync(FULL, acc, 31);
        const uint64_t head = __shfl_sync(FULL, c0, 0);
        if (head > thr) acc = warp_merge_top32(acc, c0, lane);
        g = g2;
      }
      cs.fold[0][k][p][lane] = acc;
    }
    __syncthreads();
    cur = 0;
    for (int n = P; n > 1; n >>= 1) { chain_fold_round<K, CR>(cs, cur, n, nK, warp, lane); cur ^= 1; }
    if (warp < nK) cs.keys[warp][lane] = cs.fold[cur][warp][0][lane];
  }
  if (warp == 0) { __syncwarp(); sm.keys[lane] = cs.keys[0][lane]; if (lane == 0) sm.chain_floor = cs.keys[0][KTOP - 1]; }
  {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(&cs.cls[0]);
    uint32_t* dst = reinterpret_cast<uint32_t*>(&sm.cls);
    for (uint32_t i = tid; i < sizeof(CR) / 4; i += SCAN_THREADS) dst[i] = src[i];
  }
  if (warp == SCAN_WARPS - 1) {
#pragma unroll
    for (int i = 0; i < CTLW; ++i) {
      const uint32_t idx = (uint32_t)i * 32u + lane;
      if (idx < sizeof(Ctl) / 4) reinterpret_cast<uint32_t*>(&sm.ctl)[idx] = cw[i];
    }
  }
  __syncthreads();
  if (warp == 1) {
    // shadow warp: prefetch for the first visit now, then for every chained visit as soon as warp 0 announces it
    shadow_prefetch<0>(S, sm.ctl, lane, &sm.sink, sm.keys[lane]);
    uint32_t seen = 0;
    for (;;) {
      uint32_t v;
      while ((v = *((volatile uint32_t*)&sm.chain_seq)) == seen) __nanosleep(64);
      if (v == 0xFFFFFFFFu) break;
      seen = v;
      __threadfence_block();
      shadow_prefetch<0>(S, sm.ctl, lane, &sm.sink, sm.keys[lane]);
    }
    return;
  }
  if (warp != 0) return;

  // ---------------- replay chain: warp 0 ----------------
  const uint32_t R = S.cf.R, W = S.cf.W, ncols = S.ncols;
  constexpr int CHM = 1;
  uint32_t used = 1u, kcur = 0, seq = 0;
  long long ts = t_start, tsc = t_scan;
  for (;;) {
    {
      const uint32_t n = key_node(sm.keys[lane]);
      const uint64_t* rec = S.tiles + (size_t)(n / TILE_NODES) * ((size_t)ncols * TILE_NODES) + (n % TILE_NODES);
      replay_epilogue<0, CHM>(S, sm, lane, cs.cls_id[kcur], rec, TILE_NODES, 0xFFFFFFFFu, ts, tsc);
    }
    __syncwarp();
    if (sm.ctl.done || sm.last_rescan) break;
    uint32_t nk = 0xFFFFFFFFu;
#pragma unroll
    for (int z = K - 1; z >= 0; --z) if (z < nK && !((used >> z) & 1u) && cs.cls_id[z] == sm.ctl.cur_class) nk = (uint32_t)z;
    if (nk == 0xFFFFFFFFu) break;
    const uint32_t nm = sm.nmod, nprev = sm.nmod_prev;
    if (nm + KTOP > KTOP * KB_CHAIN_MAX) break;
    ts = tsc = clock64();
    // ---- patch list nk ----
    // (1) drop the entries of modified nodes; the survivors stay sorted, so compacting them needs no sort
    uint64_t key = cs.keys[nk][lane];
    uint64_t fl = cs.keys[nk][KTOP - 1];
    bool alive = key != 0;
    if (alive) {
      const uint32_t nd = key_node(key);
      for (uint32_t i = 0; i < nm; ++i) if (sm.mod[i] == nd) { alive = false; break; }
    }
    {
      const unsigned am = __ballot_sync(FULL, alive);
      const unsigned src = __fns(am, 0, lane + 1);              // lane holding the (lane+1)-th survivor
      const uint64_t ck = __shfl_sync(FULL, key, (int)(src & 31u));
      key = src < 32u ? ck : 0ull;
    }
    // merges 32 fresh keys into the list, keeps the 32 best sorted, raises the floor to the best key dropped
    auto merge_fresh = [&](uint64_t pk) {
      pk = warp_sort_desc(pk, lane);
      const uint64_t br = __shfl_sync(FULL, pk, 31 - lane);
      const uint64_t lo = key < br ? key : br;
      uint64_t v = key > br ? key : br;
      const uint64_t dropped = warp_max_u64(lo);
      fl = dropped > fl ? dropped : fl;
#pragma unroll
      for (int j = 16; j > 0; j >>= 1) {
        const uint64_t o = __shfl_xor_sync(FULL, v, j);
        const bool take_max = (lane & j) == 0;
        v = take_max ? (o > v ? o : v) : (o < v ? o : v);
      }
      key = v;
    };
    // (2) the nodes the replay just finished modified: their current records are still in this warp's slots
    {
      uint64_t pk = 0;
      const bool mine = sm.lane_mod[lane] != 0;
      if (mine) {
        ColAcc acc{&sm.slot[sm.lane_which[lane]][0][0], (uint32_t)lane, 32u, R, W};
        pk = eval_pair(S.cf, cs.cls[nk], acc, sm.lane_node[lane], nullptr);
      }
      const unsigned cnt = __popc(__ballot_sync(FULL, mine));
      if (lane == 0) sm.ctl.pairs_replayed += (unsigned long long)cnt;
      merge_fresh(pk);
    }
    __syncwarp();
    // (3) K > 2: nodes modified by EARLIER replays of this launch (not touched again by the last one): re-read from the table
    if (K > 2) {
      for (uint32_t base = 0; base < nprev; base += 32) {
        uint64_t pk = 0;
        bool mine = base + lane < nprev;
        uint32_t nd = 0;
        if (mine) {
          nd = sm.mod[base + lane];
          for (uint32_t z = 0; z < 32; ++z) if (sm.lane_mod[z] && sm.lane_node[z] == nd) { mine = false; break; }
        }
        __syncwarp();
        if (mine) {
          const uint64_t* g = S.tiles + (size_t)(nd / TILE_NODES) * ((size_t)ncols * TILE_NODES) + (nd % TILE_NODES);
          for (uint32_t cc = 0; cc < ncols; ++cc) sm.slot[0][cc][lane] = __ldcg(g + (size_t)cc * TILE_NODES);
          ColAcc acc{&sm.slot[0][0][0], (uint32_t)lane, 32u, R, W};
          pk = eval_pair(S.cf, cs.cls[nk], acc, nd, nullptr);
        }
        const unsigned cnt = __popc(__ballot_sync(FULL, mine));
        if (lane == 0) sm.ctl.pairs_replayed += (unsigned long long)cnt;
        merge_fresh(pk);
        __syncwarp();
      }
    }
    sm.keys[lane] = key;
    if (lane == 0) { sm.chain_floor = fl; sm.ctl.chain_hits += 1; }
    {
      const uint32_t* src = reinterpret_cast<const uint32_t*>(&cs.cls[nk]);
      uint32_t* dst = reinterpret_cast<uint32_t*>(&sm.cls);
      for (uint32_t i = lane; i < sizeof(CR) / 4; i += 32) dst[i] = src[i];
    }
    used |= 1u << nk;
    kcur = nk;
    __syncwarp();
    if (lane == 0) { __threadfence_block(); *((volatile uint32_t*)&sm.chain_seq) = ++seq; }   // shadow warp: prefetch this visit
  }
  if (lane == 0) *((volatile uint32_t*)&sm.chain_seq) = 0xFFFFFFFFu;
  if (lane == 0) publish_chain(S, sm.ctl);
  __syncwarp();
  store_ctl(gctl, sm.ctl, lane);
  if (lane == 0) gctl->arrive = 0;
}

// ---------------------------------------------------------------------------------------------
// visit_overlap_kernel (single GPU): scan and replay of consecutive visits run CONCURRENTLY.
//   CTAs 0..G-1  scanners: evaluate Ctl.scan_class — the predicted class of the visit after the one being replayed —
//                over the whole table, skipping Ctl.excl (the nodes the replayer may be modifying);
//   CTA  G       replayer: consumes Ctl.list (built by the previous launch) for the current visit(s), runs the control
//                plane, writes its candidates back and contributes their fresh keys for scan_class (Ctl.patch);
//   last CTA     (ticket over G+1) merges the scan lists with the patch into Ctl.list for the next launch, and
//                publishes the next scan_class (prediction table ord_peek) and exclusion set (the new list's nodes).
// The merged list is exact for the table state at the end of the launch: every node is either scanned unmodified or
// patched from the replayer's own up-to-date copy.  A wrong prediction only costs the overlap of one launch.
// ---------------------------------------------------------------------------------------------

template <class CR = ClassRecNarrow>
__global__ void __launch_bounds__(SCAN_THREADS)
visit_overlap_kernel(const __grid_constant__ DevSession S) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  VisitSmem<CR>& sm = *reinterpret_cast<VisitSmem<CR>*>(smem_raw);
  uint64_t* tilebuf = reinterpret_cast<uint64_t*>(smem_raw + ((sizeof(VisitSmem<CR>) + 127) / 128) * 128);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  Ctl* gctl = S.ctl;
  if (*((volatile uint32_t*)&gctl->done)) return;
  const uint32_t n_scanners = gridDim.x - 1;
  const bool is_replayer = blockIdx.x == n_scanners;
  const long long t_start = clock64();

  if (!is_replayer) {
    // ---------------- scanner ----------------
    const uint32_t cls_id = *((volatile uint32_t*)&gctl->scan_class);
    if (tid == 0) { mbar_init(&sm.mbar[0], 1); mbar_init(&sm.mbar[1], 1); fence_mbar_init(); sm.n_excl = *((volatile uint32_t*)&gctl->n_excl); }
    if (tid < 32) sm.excl[tid] = *((volatile uint32_t*)&gctl->excl[tid]);
    __syncthreads();
    const uint64_t mylist = scan_phase(S, sm, tilebuf, blockIdx.x, n_scanners, cls_id, tid, lane, warp);
    if (warp == 0) S.cand[(size_t)blockIdx.x * KTOP + lane] = mylist;
  } else if (warp == 1) {
    load_ctl(sm.ctl2, gctl, lane);
    __syncwarp();
    shadow_prefetch<0>(S, sm.ctl2, lane, &sm.sink, sm.ctl2.list[lane]);
  } else if (warp == 0) {
    // ---------------- replayer ----------------
    load_ctl(sm.ctl, gctl, lane);
    __syncwarp();
    Ctl& c = sm.ctl;
    const bool go = c.list_valid != 0 && c.list_class == c.cur_class;
    if (go) {
      const uint32_t cls_id = c.list_class;
      const uint32_t patch_class = c.n_excl > 0 ? c.scan_class : 0xFFFFFFFEu;   // 0xFFFFFFFE never matches a class
      {
        const uint32_t* src = reinterpret_cast<const uint32_t*>(&class_table<CR>(S)[cls_id]);
        uint32_t* dst = reinterpret_cast<uint32_t*>(&sm.cls);
        for (uint32_t i = lane; i < sizeof(CR) / 4; i += 32) dst[i] = src[i];
      }
      sm.keys[lane] = c.list[lane];
      __syncwarp();
      if (lane == 0) c.list_valid = 0;                  // consumed
      const uint32_t n = key_node(sm.keys[lane]);
      const uint64_t* rec = S.tiles + (size_t)(n / TILE_NODES) * ((size_t)S.ncols * TILE_NODES) + (n % TILE_NODES);
      const long long t0 = clock64();
      replay_epilogue<0>(S, sm, lane, cls_id, rec, TILE_NODES, patch_class, t0, t0);
    } else if (lane == 0) c.patch_valid = 0;
    __syncwarp();
    store_ctl(gctl, c, lane);
  }

  // ---------------- ticket over scanners + replayer ----------------
  __syncthreads();
  if (warp == 0) {
    __threadfence();
    __syncwarp();
    if (lane == 0) {
      const uint32_t ticket = atomicAdd(&gctl->arrive, 1u);
      sm.is_last = (ticket == gridDim.x - 1) ? 1u : 0u;
    }
  }
  __syncthreads();
  if (!sm.is_last) return;
  __threadfence();
  const long long t_scan = clock64();

  // ---------------- merger: all 16 warps fold the scan lists; warp 0 adds the patch and publishes ----------------
  uint64_t acc = 0;
  {
    uint32_t g = warp;
    uint64_t nxt = g < n_scanners ? __ldcg(&S.cand[(size_t)g * KTOP + lane]) : 0ull;
    while (g < n_scanners) {
      const uint64_t cur = nxt;
      const uint32_t g2 = g + SCAN_WARPS;
      nxt = g2 < n_scanners ? __ldcg(&S.cand[(size_t)g2 * KTOP + lane]) : 0ull;
      const uint64_t thr = __shfl_sync(FULL, acc, 31);
      const uint64_t head = __shfl_sync(FULL, cur, 0);
      if (head > thr) acc = warp_merge_top32(acc, cur, lane);
      g = g2;
    }
    acc = cta_fold_lists(acc, sm.wlist, warp, lane);
  }
  if (warp != 0) return;
  load_ctl(sm.ctl, gctl, lane);
  __syncwarp();
  Ctl& c = sm.ctl;
  const uint32_t n_excl0 = c.n_excl, scan_class0 = c.scan_class;
  if (c.patch_valid) acc = warp_merge_top32(acc, c.patch[lane], lane);
  __syncwarp();
  c.list[lane] = acc;
  const unsigned nz = __ballot_sync(FULL, acc != 0);
  if (lane == 0) {
    c.list_class = scan_class0;
    c.list_valid = (n_excl0 == 0 || c.patch_valid) ? 1u : 0u;
    c.scans += 1; c.pairs_scanned += (unsigned long long)S.N;
    if (n_excl0 > 0) { c.predictions += 1; if (!c.patch_valid) c.mispredictions += 1; }
  }
  __syncwarp();
  if (!c.done) {
    const bool useful = c.list_valid != 0 && c.list_class == c.cur_class;
    if (useful) {
      c.excl[lane] = acc ? key_node(acc) : 0u;
      if (lane == 0) {
        const uint32_t pk = S.ord_peek[S.job_pos[(uint32_t)c.cur_job]];
        c.scan_class = pk != 0xFFFFFFFFu ? pk : c.cur_class;
        c.n_excl = (uint32_t)__popc(nz);
      }
    } else if (lane == 0) { c.scan_class = c.cur_class; c.n_excl = 0; }
  }
  __syncwarp();
  if (lane == 0) {
    const long long t_end = clock64();
    c.cyc_scan += (unsigned long long)(t_scan - t_start);
    c.cyc_merge += (unsigned long long)(t_end - t_scan);
    c.cyc_total += (unsigned long long)(t_end - t_start);
  }
  __syncwarp();
  store_ctl(gctl, c, lane);
  __syncwarp();
  if (lane == 0) gctl->arrive = 0;
}

// ---------------------------------------------------------------------------------------------
// replay_kernel (sharded node axis only): one warp merges the ranks' all-gathered candidate lists, each
// lane finds the record of its candidate in the owning rank's block and the shared epilogue replays.
// Every rank runs this identically on identical inputs, so every replica applies the same updates.
// ---------------------------------------------------------------------------------------------
template <int BF>
__global__ void __launch_bounds__(64)
replay_kernel(const __grid_constant__ DevSession S) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  VisitSmem<>& sm = *reinterpret_cast<VisitSmem<>*>(smem_raw);      // narrow sessions only: the sharded path takes R <= KB_NARROW_R, W <= KB_NARROW_W
  const int lane = threadIdx.x & 31;
  Ctl* gctl = S.ctl;
  if (*((volatile uint32_t*)&gctl->done)) return;
  if (threadIdx.x >= 32) {                       // warp 1: shadow prefetch from its own copy of the control block
    load_ctl(sm.ctl2, gctl, lane);
    __syncwarp();
    shadow_prefetch<BF>(S, sm.ctl2, lane, &sm.sink, 0ull);
    return;
  }
  const uint32_t cls_id = *((volatile uint32_t*)&gctl->cur_class);
  {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(&S.classes[cls_id]);
    uint32_t* dst = reinterpret_cast<uint32_t*>(&sm.cls);
    for (uint32_t i = lane; i < sizeof(ClassRec) / 4; i += 32) dst[i] = src[i];
  }
  const long long t_start = clock64();
  const size_t rank_u64 = (size_t)xchg_u64(S.ncols);
  if (BF) {
    uint32_t f = (uint32_t)lane < S.world ? (uint32_t)__ldcg(S.recvbuf + (size_t)lane * rank_u64 + (size_t)(1 + S.ncols) * 32) : 0u;
    f = __reduce_or_sync(FULL, f);
    if (lane == 0) sm.pred_any_all = f;
    __syncwarp();
  }
  uint64_t acc = __ldcg(S.recvbuf + lane);
  for (uint32_t r = 1; r < S.world; ++r) acc = warp_merge_top32(acc, __ldcg(S.recvbuf + r * rank_u64 + lane), lane);
  sm.keys[lane] = acc;
  const uint32_t node = key_node(acc);
  uint32_t owner = node / S.nodes_per_rank;
  owner = owner < S.world ? owner : S.world - 1;
  uint32_t idx = 0;
  if (acc)
    for (uint32_t i = 0; i < 32; ++i)
      if (__ldcg(S.recvbuf + owner * rank_u64 + i) == acc) idx = i;
  if (lane == 0) sm.ctl = *gctl;
  __syncwarp();
  replay_epilogue<BF>(S, sm, lane, cls_id, S.recvbuf + owner * rank_u64 + 32 + idx, 32u, 0xFFFFFFFFu, t_start, clock64());
  store_ctl(gctl, sm.ctl, lane);
  if (lane == 0) gctl->arrive = 0;
}

// ---------------------------------------------------------------------------------------------
// K4: gang commit.  One warp per job: inclusive prefix scan of the Allocated flags over the job's
// tasks in processing order; e* = first Allocate at which ReadyTaskNum >= MinAvailable (always, when
// gang's JobReadyFn is not enabled); a task allocated at position i is dispatched at step[max(i, e*)].
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
gang_commit_kernel(const __grid_constant__ DevSession S, const int32_t* __restrict__ job_ready0,
                   const uint32_t* __restrict__ bf_ord_task, const uint32_t* __restrict__ bf_job_ord_off,
                   const uint32_t* __restrict__ bf_job_pos) {
  const uint32_t warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp_global >= S.J) return;
  const uint32_t j = warp_global;
  // processed slots in step order: the allocate view's, then the backfill view's (backfill runs after allocate)
  const uint32_t lo = S.job_ord_off[j], na = S.job_pos[j] - lo;
  const uint32_t blo = bf_job_ord_off[j], nb = bf_job_pos[j] - blo;
  const uint32_t n = na + nb;
  if (n == 0) return;
  auto task_at = [&](uint32_t v) { return v < na ? S.ord_task[lo + v] : bf_ord_task[blo + (v - na)]; };
  // a best-effort task the backfill pass went through without finding a node is no longer "skipped"
  for (uint32_t v = na + lane; v < n; v += 32) {
    const uint32_t t = task_at(v);
    if (S.dec[t].kind == KB_KIND_SKIPPED) S.dec[t].kind = KB_KIND_NONE;
  }
  __syncwarp();
  const int32_t need = S.gang_ready ? S.job_min_avail[j] - job_ready0[j] : 0;   // allocations required before JobReady
  // pass 1: find e* (slot index) and its step.  A phantom (backfill: Allocated on no node, step none) counts towards
  // ReadyTaskNum but its ssn.Allocate returned before the JobReady check, so e* is always a REAL allocation.
  uint32_t estar = 0xFFFFFFFFu, estep = 0;
  int32_t carried = 0;
  bool phantoms = false;
  for (uint32_t base = 0; base < n && estar == 0xFFFFFFFFu; base += 32) {
    const uint32_t i = base + lane;
    uint32_t alloc = 0, step = 0xFFFFFFFFu;
    if (i < n) { const kb_decision d = S.dec[task_at(i)]; alloc = d.kind == KB_KIND_ALLOCATED; step = d.step; }
    const bool real = alloc && step != 0xFFFFFFFFu;
    phantoms = phantoms || __any_sync(FULL, alloc && !real);
    int32_t x = (int32_t)alloc;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { int32_t y = __shfl_up_sync(FULL, x, o); if (lane >= o) x += y; }
    const int32_t incl = carried + x;
    const unsigned m = __ballot_sync(FULL, real && incl >= need);
    if (m) {
      const int src = __ffs(m) - 1;
      estar = base + src;
      estep = __shfl_sync(FULL, step, src);
    }
    carried = __shfl_sync(FULL, incl, 31);
  }
  if (estar == 0xFFFFFFFFu) return;                   // never became ready: nothing is dispatched
  for (uint32_t i = lane; i < n; i += 32) {
    const uint32_t t = task_at(i);
    kb_decision d = S.dec[t];
    if (d.kind != KB_KIND_ALLOCATED) continue;
    if (i <= estar) { d.dispatched = 1; d.dispatch_step = estep; }
    else if (d.step != 0xFFFFFFFFu) { d.dispatched = 1; d.dispatch_step = d.step; }
    else {
      // a phantom after e*: the next successful ssn.Allocate of the job finds it in TaskStatusIndex[Allocated] and
      // dispatches it (session.go:277-285); if there is none it stays undispatched
      for (uint32_t k = i + 1; k < n; ++k) {
        const kb_decision dk = S.dec[task_at(k)];
        if (dk.kind == KB_KIND_ALLOCATED && dk.step != 0xFFFFFFFFu) { d.dispatched = 1; d.dispatch_step = dk.step; break; }
      }
      if (!d.dispatched) continue;
    }
    S.dec[t] = d;
  }
}

// kb_backfill: the backfill view continues the allocate view's Allocate sequence numbers and cycle counters
// (`carry` = kb_allocate ran on this session state; otherwise backfill is the first action and starts from zero)
__global__ void seed_backfill_kernel(const Ctl* __restrict__ main_ctl, Ctl* __restrict__ bf, const int carry) {
  if (threadIdx.x != 0 || bf->bf_seeded) return;
  bf->bf_seeded = 1;
  if (!carry) return;
  bf->step = main_ctl->step;
  bf->tasks_processed = main_ctl->tasks_processed; bf->tasks_allocated = main_ctl->tasks_allocated;
  bf->tasks_pipelined = main_ctl->tasks_pipelined; bf->visits = main_ctl->visits;
  bf->scans = main_ctl->scans; bf->rescans = main_ctl->rescans;
  bf->pairs_logical = main_ctl->pairs_logical; bf->pairs_scanned = main_ctl->pairs_scanned; bf->pairs_replayed = main_ctl->pairs_replayed;
  bf->cyc_scan = main_ctl->cyc_scan; bf->cyc_merge = main_ctl->cyc_merge; bf->cyc_replay = main_ctl->cyc_replay;
  bf->cyc_total = main_ctl->cyc_total; bf->cyc_steps = main_ctl->cyc_steps; bf->cyc_ctl = main_ctl->cyc_ctl;
  bf->predictions = main_ctl->predictions; bf->mispredictions = main_ctl->mispredictions;
}

// ---------------------------------------------------------------------------------------------
// Full matrix for tasks [task_lo, task_hi) x all nodes (parity / debug).
// grid = (NT, task chunks); each CTA stages one node tile with TMA and walks its task chunk.
// ---------------------------------------------------------------------------------------------
constexpr int MATRIX_TASKS_PER_CTA = 32;

template <class CR = ClassRecNarrow>
__global__ void __launch_bounds__(MATRIX_THREADS)
matrix_kernel(const __grid_constant__ DevSession S, const uint32_t* __restrict__ task_class, uint32_t task_lo, uint32_t task_hi,
              uint8_t* __restrict__ fit, double* __restrict__ score) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ CR cls;
  __shared__ uint64_t mbar;
  uint64_t* tilebuf = reinterpret_cast<uint64_t*>(smem_raw);
  const int tid = threadIdx.x;
  const uint32_t tile_u64 = S.ncols * TILE_NODES;
  if (tid == 0) {
    mbar_init(&mbar, 1); fence_mbar_init();
    mbar_expect_tx(&mbar, tile_u64 * 8u);
    tma_load_1d(tilebuf, S.tiles + (size_t)blockIdx.x * tile_u64, tile_u64 * 8u, &mbar);
  }
  __syncthreads();
  mbar_wait(&mbar, 0);
  const uint32_t node = blockIdx.x * TILE_NODES + tid;
  const uint32_t t0 = task_lo + blockIdx.y * MATRIX_TASKS_PER_CTA;
  const uint32_t t1 = min(task_hi, t0 + MATRIX_TASKS_PER_CTA);
  ColAcc acc{tilebuf, (uint32_t)tid, TILE_NODES, S.cf.R, S.cf.W};
  for (uint32_t t = t0; t < t1; ++t) {
    __syncthreads();
    {
      const uint32_t* src = reinterpret_cast<const uint32_t*>(&class_table<CR>(S)[task_class[t]]);
      uint32_t* dst = reinterpret_cast<uint32_t*>(&cls);
      for (uint32_t i = tid; i < sizeof(CR) / 4; i += MATRIX_THREADS) dst[i] = src[i];
    }
    __syncthreads();
    if (node < S.N) {
      uint64_t key = eval_pair(S.cf, cls, acc, node, nullptr);
      // inter-pod affinity sessions on the counter path: predicate step 10 against the CURRENT counters (the priority terms need
      // reductions over the feasible nodes: kb_predicate_score returns fit only for such classes)
      if (key && S.aff.on && S.cf.predicates && !aff_pred(S.aff, S.aff.cls[task_class[t]], S.N, node)) key = 0;
      const size_t o = (size_t)(t - task_lo) * S.N + node;
      if (fit) fit[o] = key != 0;
      if (score) score[o] = key ? (double)(key_score(key) - S.cf.score_bias) : 0.0;
    }
  }
}

// K1+K2+K3 fused: per-task best packed key over ALL nodes in one launch.
template <class CR = ClassRecNarrow>
__global__ void __launch_bounds__(MATRIX_THREADS)
best_nodes_kernel(const __grid_constant__ DevSession S, const uint32_t* __restrict__ task_class, uint32_t task_lo, uint32_t task_hi,
                  unsigned long long* __restrict__ best_key) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ CR cls;
  __shared__ uint64_t mbar;
  uint64_t* tilebuf = reinterpret_cast<uint64_t*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31;
  const uint32_t tile_u64 = S.ncols * TILE_NODES;
  if (tid == 0) {
    mbar_init(&mbar, 1); fence_mbar_init();
    mbar_expect_tx(&mbar, tile_u64 * 8u);
    tma_load_1d(tilebuf, S.tiles + (size_t)blockIdx.x * tile_u64, tile_u64 * 8u, &mbar);
  }
  __syncthreads();
  mbar_wait(&mbar, 0);
  const uint32_t node = blockIdx.x * TILE_NODES + tid;
  const uint32_t chunk = (task_hi - task_lo + gridDim.y - 1) / gridDim.y;
  const uint32_t t0 = task_lo + blockIdx.y * chunk;
  const uint32_t t1 = min(task_hi, t0 + chunk);
  ColAcc acc{tilebuf, (uint32_t)tid, TILE_NODES, S.cf.R, S.cf.W};
  uint32_t cur_cls = 0xFFFFFFFFu;
  for (uint32_t t = t0; t < t1; ++t) {
    const uint32_t cid = task_class[t];
    if (cid != cur_cls) {            // tasks of a PodGroup share a class: reload only on change (uniform branch)
      __syncthreads();
      const uint32_t* src = reinterpret_cast<const uint32_t*>(&class_table<CR>(S)[cid]);
      uint32_t* dst = reinterpret_cast<uint32_t*>(&cls);
      for (uint32_t i = tid; i < sizeof(CR) / 4; i += MATRIX_THREADS) dst[i] = src[i];
      __syncthreads();
      cur_cls = cid;
    }
    uint64_t key = node < S.N ? eval_pair(S.cf, cls, acc, node, nullptr) : 0ull;
    key = warp_max_u64(key);
    if (lane == 0 && key) atomicMax(&best_key[t - task_lo], (unsigned long long)key);
  }
}

}  // namespace kb
