// kb_evict_kernels.cu — reclaim / preempt on the device (kb_evict.h holds the algorithm, shared with the CPU emulation).
//
// evict_kernel<PREEMPT>   cooperative grid: W worker CTAs + 1 master CTA.
//   master  ONE thread runs the action exactly as written in kb_evict.h (queue / job heaps with Go's container/heap semantics,
//           Statement commit / discard, the serial commit on the chosen node).  Whenever a preemptor needs its pass over the
//           node table it writes the preemptor + its class into the mailbox, posts a command word (release) and waits for the
//           workers' arrival counter; preemptors whose sweep is known to fail (same class, same filter, unchanged state) never
//           leave the master thread.
//   worker  CTAs poll the command word (acquire), sweep their share of the nodes — one node per thread per iteration: K1
//           predicate, K2 score for preempt, the serial victim walk of the node's Running tasks — reduce the packed keys
//           (warp REDUX, one 64-bit atomicMax per CTA) and arrive.
//   pass 1  a preempting class with preferred node-affinity terms (evict_pref) takes one more round trip through the same mailbox
//           before its sweep: the workers reduce the NodeAffinityPriority max count over all their nodes (warp REDUX.MAX, one
//           atomicMax per CTA into EvictCtl.pmax) and arrive; the sweep command that follows reads pmax from the mailbox.  Workers
//           keep the class's ClassPref in shared memory and copy it only when the class changes.
//   passes 2-4  a preempting class with an inter-pod weight list (evict_aff, InterPodAffinityPriority) takes three round trips
//           instead: 2 clears AffDev.dom_sum, 3 adds the weights of the pods on every node that passes ssn.PredicateFn to their
//           domains (64-bit integer atomicAdd: the sums do not depend on the order), 4 reduces the min / max count over the same
//           nodes (warp REDUX on both halves, one atomicMin / atomicMax per CTA into EvictCtl.amin / amax) and, for a class that
//           also has preferred node-affinity terms, pmax in the same pass.  Classes without a list post exactly what they did before.
//
// Coherence: the master mutates node records, job / queue accounting and the Running tasks' states between two sweeps.  It
// publishes them with a release store of the command word; thread 0 of every worker CTA reads that word with ld.acquire.gpu —
// which invalidates the SM's L1 — before the CTA barrier that starts the sweep, so the workers' ordinary (L1-cached) loads see
// the current tables, and nothing changes while a sweep runs.  The master's own acquire on the arrival counter does the same
// for the workers' error word.
#include <cuda_runtime.h>

#include "kb_evict.h"
#include "kb_evict_launch.h"

namespace kb {

constexpr int EVICT_THREADS = 512;
constexpr uint32_t EVICT_EXIT = 0xFFFFFFFFu;
static_assert(std::is_same<ClassRec, ClassRecNarrow>::value, "RecKind::Own runs the kernels' default (narrow) instances");

__device__ __forceinline__ uint32_t ev_ld_acquire(const uint32_t* p) {
  uint32_t v; asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ void ev_st_release(uint32_t* p, uint32_t v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// min / max of a signed 64-bit value over the warp with two 32-bit REDUX each: the high words (signed), then the low words
// (unsigned) of the lanes that hold the winning high word
__device__ __forceinline__ long long ev_warp_max(const long long v) {
  const int hi = (int)(v >> 32);
  const unsigned lo = (unsigned)v;
  const int mhi = __reduce_max_sync(0xFFFFFFFFu, hi);
  const unsigned mlo = __reduce_max_sync(0xFFFFFFFFu, hi == mhi ? lo : 0u);
  return (long long)(((unsigned long long)(unsigned)mhi << 32) | mlo);
}
__device__ __forceinline__ long long ev_warp_min(const long long v) {
  const int hi = (int)(v >> 32);
  const unsigned lo = (unsigned)v;
  const int mhi = __reduce_min_sync(0xFFFFFFFFu, hi);
  const unsigned mlo = __reduce_min_sync(0xFFFFFFFFu, hi == mhi ? lo : 0xFFFFFFFFu);
  return (long long)(((unsigned long long)(unsigned)mhi << 32) | mlo);
}

// the master thread's Exec: single-threaded control, the sweep is farmed out.  CR: class record type of the session (ClassRecT),
// the type of the mailbox record (EvictCtl.cls / cls_wide / cls_atoms) and of the workers' copy
template <class CR>
struct MasterExec {
  EvictCtl* g;
  uint32_t seq;
  __device__ __forceinline__ int tid() const { return 0; }
  __device__ __forceinline__ int nthreads() const { return 1; }
  __device__ __forceinline__ void sync() {}
  __device__ __forceinline__ uint32_t bcast(uint32_t v) { return v; }
  __device__ __forceinline__ bool jobs_scanned() const { return true; }      // evict_scan_kernel ran before this kernel
  __device__ __forceinline__ void clear_max() {}
  __device__ __forceinline__ CR& cls() {
    if constexpr (std::is_same<CR, ClassRec>::value) return g->cls;
    else if constexpr (std::is_same<CR, ClassRecWide>::value) return g->cls_wide;
    else return g->cls_atoms;
  }
  __device__ __forceinline__ Preemptor& pre() { return g->pre; }
  __device__ __forceinline__ void post(const uint32_t pass) {     // one command to every worker CTA, back when all have arrived
    g->pass = pass;
    g->arrived = 0u;
    __threadfence();                                 // the mailbox (pre, cls, pmax) and every table write of earlier commits are visible first
    seq += 1;
    ev_st_release(&g->cmd_seq, seq);
    const uint32_t nw = g->n_workers;
    while (ev_ld_acquire(&g->arrived) < nw) __nanosleep(40);
  }
  __device__ __forceinline__ uint64_t sweep(const DevSession& S, const EvictDev&, const Preemptor& P, const CR&) {
    // preferred node-affinity terms: pass 1 leaves the max count in g->pmax, which is then the sweep's normalisation.  It is
    // taken afresh for every sweep: a Pipeline raises a node's pod count, and max_pods can drop that node together with its count.
    // inter-pod weight list: clear dom_sum, fill it, reduce min / max (and pmax in the same pass) — three commands.
    if (evict_aff(S, P)) { post(2u); post(3u); g->amin = 0ll; g->amax = 0ll; g->pmax = 0u; post(4u); }
    else if (evict_pref<CR>(S, P)) { g->pmax = 0u; post(1u); }
    g->red = 0ull;
    post(0u);
    return *((volatile unsigned long long*)&g->red);
  }
};

template <int PREEMPT, class CR = ClassRecNarrow>
__global__ void __launch_bounds__(EVICT_THREADS, 1)
evict_kernel(const __grid_constant__ DevSession S, const __grid_constant__ EvictDev E) {
  EvictCtl* g = E.ctl;
  if (blockIdx.x == gridDim.x - 1) {
    // ---------------- master ----------------
    if (threadIdx.x != 0) return;
    MasterExec<CR> x{g, 0u};
    if (PREEMPT) run_preempt(x, S, E);
    else run_reclaim(x, S, E);
    __threadfence();
    ev_st_release(&g->cmd_seq, EVICT_EXIT);
    return;
  }
  // ---------------- workers ----------------
  __shared__ CR s_cls;
  __shared__ Preemptor s_pre;
  __shared__ ClassPrefOf<CR> s_pref;                     // preferred node-affinity terms of class s_pref_cls
  __shared__ ClassAff s_aff;                       // inter-pod weight list record of class s_aff_cls
  __shared__ uint64_t s_red[EVICT_THREADS / 32];
  __shared__ long long s_mn[EVICT_THREADS / 32], s_mx[EVICT_THREADS / 32];
  __shared__ uint32_t s_list[EVICT_THREADS];       // pass 3: each warp's nodes that pass ssn.PredicateFn, compacted
  __shared__ long long s_amin, s_amax;
  __shared__ uint32_t s_cmd, s_err, s_pass, s_pmax, s_pref_cls, s_aff_cls;
  const uint32_t nw = gridDim.x - 1;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t seen = 0;
  if (threadIdx.x == 0) { s_pref_cls = 0xFFFFFFFFu; s_aff_cls = 0xFFFFFFFFu; }
  for (;;) {
    if (threadIdx.x == 0) {
      uint32_t v;
      while ((v = ev_ld_acquire(&g->cmd_seq)) == seen) __nanosleep(40);
      s_cmd = v; s_err = 0;
      s_pass = *((volatile uint32_t*)&g->pass); s_pmax = *((volatile uint32_t*)&g->pmax);
      s_amin = *((volatile long long*)&g->amin); s_amax = *((volatile long long*)&g->amax);
    }
    __syncthreads();
    const uint32_t cmd = s_cmd;
    if (cmd == EVICT_EXIT) return;
    seen = cmd;
    {
      const uint32_t* src = reinterpret_cast<const uint32_t*>(&g->cls);
      uint32_t* dst = reinterpret_cast<uint32_t*>(&s_cls);
      for (uint32_t i = threadIdx.x; i < sizeof(CR) / 4; i += EVICT_THREADS) dst[i] = src[i];
      const uint32_t* ps = reinterpret_cast<const uint32_t*>(&g->pre);
      uint32_t* pd = reinterpret_cast<uint32_t*>(&s_pre);
      for (uint32_t i = threadIdx.x; i < sizeof(Preemptor) / 4; i += EVICT_THREADS) pd[i] = ps[i];
    }
    __syncthreads();
    const ClassPrefOf<CR>* cp = evict_pref<CR>(S, s_pre);    // uniform across the CTA
    if (cp && s_pref_cls != s_pre.cls) {           // 160 B (544 B with 16 words), only when the class changes
      const uint32_t* src = reinterpret_cast<const uint32_t*>(cp);
      uint32_t* dst = reinterpret_cast<uint32_t*>(&s_pref);
      for (uint32_t i = threadIdx.x; i < sizeof(ClassPrefOf<CR>) / 4; i += EVICT_THREADS) dst[i] = src[i];
      __syncthreads();
      if (threadIdx.x == 0) s_pref_cls = s_pre.cls;
    }
    const ClassAff* ca = evict_aff(S, s_pre);       // uniform across the CTA
    if (ca && s_aff_cls != s_pre.cls) {             // 72 B, only when the class changes
      const uint32_t* src = reinterpret_cast<const uint32_t*>(ca);
      uint32_t* dst = reinterpret_cast<uint32_t*>(&s_aff);
      for (uint32_t i = threadIdx.x; i < sizeof(ClassAff) / 4; i += EVICT_THREADS) dst[i] = src[i];
      __syncthreads();
      if (threadIdx.x == 0) s_aff_cls = s_pre.cls;
    }
    if (s_pass == 2u || s_pass == 3u) {
      if (s_pass == 2u) {                          // clear the weights per domain
        for (uint32_t i = blockIdx.x * EVICT_THREADS + threadIdx.x; i < S.aff.dom_total; i += nw * EVICT_THREADS) S.aff.dom_sum[i] = 0;
      } else {
        // weights per domain (aff_pass1_node) over the nodes that pass ssn.PredicateFn: each thread tests one node, the warp
        // compacts its passing nodes and spreads (node, weight entry) pairs over the lanes — a class can weigh hundreds of kinds
        const uint32_t wc = s_aff.w_cnt;
        uint32_t* list = s_list + warp * 32;
        auto add = [&](uint32_t slot, long long v) { atomicAdd(reinterpret_cast<unsigned long long*>(&S.aff.dom_sum[slot]), (unsigned long long)v); };
        for (uint32_t n0 = blockIdx.x * EVICT_THREADS + (uint32_t)warp * 32u; n0 < S.N; n0 += nw * EVICT_THREADS) {
          const uint32_t n = n0 + (uint32_t)lane;
          const bool ok = n < S.N && evict_pred_ok(S, s_cls, n);
          const unsigned m = __ballot_sync(0xFFFFFFFFu, ok);
          if (ok) list[__popc(m & ((1u << lane) - 1u))] = n;
          __syncwarp();
          const uint32_t items = (uint32_t)__popc(m) * wc;
          for (uint32_t k = (uint32_t)lane; k < items; k += 32u) aff_pass1_node(S.aff, s_aff, S.N, list[k / wc], add, k % wc, wc);
          __syncwarp();
        }
      }
      __threadfence();
      __syncthreads();
      if (threadIdx.x == 0) atomicAdd(&g->arrived, 1u);
      continue;
    }
    if (s_pass == 4u) {                            // min / max InterPodAffinityPriority count (+ NodeAffinityPriority max) over this CTA's nodes
      long long mn = 0, mx = 0;
      uint32_t pm = 0;
      for (uint32_t n = blockIdx.x * EVICT_THREADS + threadIdx.x; n < S.N; n += nw * EVICT_THREADS) {
        if (!evict_pred_ok(S, s_cls, n)) continue;
        const long long c = aff_count_node(S.aff, s_aff, S.N, n);
        mn = c < mn ? c : mn; mx = c > mx ? c : mx;
        if (cp) { const uint32_t v = evict_pref_count(S, s_cls, s_pref, n); pm = v > pm ? v : pm; }
      }
      mn = ev_warp_min(mn); mx = ev_warp_max(mx);
      pm = __reduce_max_sync(0xFFFFFFFFu, pm);
      if (lane == 0) { s_mn[warp] = mn; s_mx[warp] = mx; s_red[warp] = pm; }
      __syncthreads();
      if (warp == 0) {
        const long long a = ev_warp_min(lane < EVICT_THREADS / 32 ? s_mn[lane] : 0ll);
        const long long b = ev_warp_max(lane < EVICT_THREADS / 32 ? s_mx[lane] : 0ll);
        const uint32_t p = __reduce_max_sync(0xFFFFFFFFu, lane < EVICT_THREADS / 32 ? (uint32_t)s_red[lane] : 0u);
        if (lane == 0) {
          if (a < 0) atomicMin(&g->amin, a);       // both start at 0 (interpod_affinity.go:205-214)
          if (b > 0) atomicMax(&g->amax, b);
          if (p) atomicMax(&g->pmax, p);
          __threadfence();
          atomicAdd(&g->arrived, 1u);
        }
      }
      __syncthreads();
      continue;
    }
    if (s_pass == 1u) {                            // pass 1: max NodeAffinityPriority count over this CTA's nodes
      uint32_t m = 0;
      for (uint32_t n = blockIdx.x * EVICT_THREADS + threadIdx.x; n < S.N; n += nw * EVICT_THREADS) {
        const uint32_t v = evict_pref_count(S, s_cls, s_pref, n);
        m = v > m ? v : m;
      }
      m = __reduce_max_sync(0xFFFFFFFFu, m);
      if (lane == 0) s_red[warp] = m;
      __syncthreads();
      if (warp == 0) {
        const uint32_t x = __reduce_max_sync(0xFFFFFFFFu, lane < EVICT_THREADS / 32 ? (uint32_t)s_red[lane] : 0u);
        if (lane == 0) {
          if (x) atomicMax(&g->pmax, x);
          __threadfence();
          atomicAdd(&g->arrived, 1u);
        }
      }
      __syncthreads();
      continue;
    }
    uint64_t best = 0;
    uint32_t err = 0;
    const EvictPrioT<CR> pr{cp ? &s_pref : nullptr, s_pmax, ca ? &s_aff : nullptr, s_amin, s_amax};
    for (uint32_t n = blockIdx.x * EVICT_THREADS + threadIdx.x; n < S.N; n += nw * EVICT_THREADS) {
      const uint64_t k = evict_node_key(S, E, s_pre, s_cls, pr, n, &err);
      best = k > best ? k : best;
    }
    if (err) s_err = err;
    {
      const unsigned hi = (unsigned)(best >> 32), lo = (unsigned)best;
      const unsigned mhi = __reduce_max_sync(0xFFFFFFFFu, hi);
      const unsigned mlo = __reduce_max_sync(0xFFFFFFFFu, hi == mhi ? lo : 0u);
      if (lane == 0) s_red[warp] = ((uint64_t)mhi << 32) | mlo;
    }
    __syncthreads();
    if (warp == 0) {
      const uint64_t r = lane < EVICT_THREADS / 32 ? s_red[lane] : 0ull;
      const unsigned rh = (unsigned)(r >> 32), rl = (unsigned)r;
      const unsigned xh = __reduce_max_sync(0xFFFFFFFFu, rh);
      const unsigned xl = __reduce_max_sync(0xFFFFFFFFu, rh == xh ? rl : 0u);
      if (lane == 0) {
        if (xh | xl) atomicMax(&g->red, ((unsigned long long)xh << 32) | xl);
        if (s_err) g->error = s_err;
        __threadfence();
        atomicAdd(&g->arrived, 1u);
      }
    }
    __syncthreads();      // s_cls / s_pre / s_red are reused by the next command
  }
}

// evict_init's per-job scan (WaitingTaskNum, first Pending task, the job's Allocated members into the atom counts), one thread per job
template <class CR = ClassRecNarrow>
__global__ void evict_scan_kernel(const __grid_constant__ DevSession S, const __grid_constant__ EvictDev E) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < S.J) evict_scan_job<CR>(S, E, j);
}

cudaError_t launch_evict(const bool preempt, const DevSession& S, const EvictDev& E, const int sm_count, cudaStream_t stream) {
  // workers: one node per thread per sweep iteration, at most one CTA per SM next to the master's (co-residency: they spin)
  int workers = (int)((S.N + EVICT_THREADS - 1) / EVICT_THREADS);
  workers = workers < 1 ? 1 : (workers > sm_count - 1 ? sm_count - 1 : workers);
  if (workers < 1) workers = 1;
  cudaError_t c = cudaMemcpyAsync(reinterpret_cast<char*>(E.ctl) + offsetof(EvictCtl, n_workers), &workers, 4, cudaMemcpyHostToDevice, stream);
  if (c != cudaSuccess) return c;
  c = cudaMemsetAsync(reinterpret_cast<char*>(E.ctl) + offsetof(EvictCtl, cmd_seq), 0, 8, stream);      // cmd_seq, arrived
  if (c != cudaSuccess) return c;
  c = cudaMemsetAsync(reinterpret_cast<char*>(E.ctl) + offsetof(EvictCtl, cls_valid), 0, 4, stream);
  if (c != cudaSuccess) return c;
  DevSession s = S; EvictDev ev = E;
  void* args[] = {(void*)&s, (void*)&ev};
  return with_rec(rec_kind(S.cf.R, S.cf.W), [&](auto t) {
    using CR = typename decltype(t)::type;
    if (S.J) evict_scan_kernel<CR><<<(S.J + 255) / 256, 256, 0, stream>>>(S, E);
    const void* fn = preempt ? (const void*)evict_kernel<1, CR> : (const void*)evict_kernel<0, CR>;
    return cudaLaunchCooperativeKernel(fn, dim3(workers + 1), dim3(EVICT_THREADS), args, 0, stream);
  });
}

}  // namespace kb
