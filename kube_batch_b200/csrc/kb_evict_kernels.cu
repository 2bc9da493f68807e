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

__device__ __forceinline__ uint32_t ev_ld_acquire(const uint32_t* p) {
  uint32_t v; asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ void ev_st_release(uint32_t* p, uint32_t v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// the master thread's Exec: single-threaded control, the sweep is farmed out
struct MasterExec {
  EvictCtl* g;
  uint32_t seq;
  __device__ __forceinline__ int tid() const { return 0; }
  __device__ __forceinline__ int nthreads() const { return 1; }
  __device__ __forceinline__ void sync() {}
  __device__ __forceinline__ uint32_t bcast(uint32_t v) { return v; }
  __device__ __forceinline__ bool jobs_scanned() const { return true; }      // evict_scan_kernel ran before this kernel
  __device__ __forceinline__ void clear_max() {}
  __device__ __forceinline__ ClassRec& cls() { return g->cls; }
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
  __device__ __forceinline__ uint64_t sweep(const DevSession& S, const EvictDev&, const Preemptor& P, const ClassRec&) {
    // preferred node-affinity terms: pass 1 leaves the max count in g->pmax, which is then the sweep's normalisation.  It is
    // taken afresh for every sweep: a Pipeline raises a node's pod count, and max_pods can drop that node together with its count.
    if (evict_pref(S, P)) { g->pmax = 0u; post(1u); }
    g->red = 0ull;
    post(0u);
    return *((volatile unsigned long long*)&g->red);
  }
};

template <int PREEMPT>
__global__ void __launch_bounds__(EVICT_THREADS, 1)
evict_kernel(const __grid_constant__ DevSession S, const __grid_constant__ EvictDev E) {
  EvictCtl* g = E.ctl;
  if (blockIdx.x == gridDim.x - 1) {
    // ---------------- master ----------------
    if (threadIdx.x != 0) return;
    MasterExec x{g, 0u};
    if (PREEMPT) run_preempt(x, S, E);
    else run_reclaim(x, S, E);
    __threadfence();
    ev_st_release(&g->cmd_seq, EVICT_EXIT);
    return;
  }
  // ---------------- workers ----------------
  __shared__ ClassRec s_cls;
  __shared__ Preemptor s_pre;
  __shared__ ClassPref s_pref;                     // preferred node-affinity terms of class s_pref_cls
  __shared__ uint64_t s_red[EVICT_THREADS / 32];
  __shared__ uint32_t s_cmd, s_err, s_pass, s_pmax, s_pref_cls;
  const uint32_t nw = gridDim.x - 1;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t seen = 0;
  if (threadIdx.x == 0) s_pref_cls = 0xFFFFFFFFu;
  for (;;) {
    if (threadIdx.x == 0) {
      uint32_t v;
      while ((v = ev_ld_acquire(&g->cmd_seq)) == seen) __nanosleep(40);
      s_cmd = v; s_err = 0;
      s_pass = *((volatile uint32_t*)&g->pass); s_pmax = *((volatile uint32_t*)&g->pmax);
    }
    __syncthreads();
    const uint32_t cmd = s_cmd;
    if (cmd == EVICT_EXIT) return;
    seen = cmd;
    {
      const uint32_t* src = reinterpret_cast<const uint32_t*>(&g->cls);
      uint32_t* dst = reinterpret_cast<uint32_t*>(&s_cls);
      for (uint32_t i = threadIdx.x; i < sizeof(ClassRec) / 4; i += EVICT_THREADS) dst[i] = src[i];
      const uint32_t* ps = reinterpret_cast<const uint32_t*>(&g->pre);
      uint32_t* pd = reinterpret_cast<uint32_t*>(&s_pre);
      for (uint32_t i = threadIdx.x; i < sizeof(Preemptor) / 4; i += EVICT_THREADS) pd[i] = ps[i];
    }
    __syncthreads();
    const ClassPref* cp = evict_pref(S, s_pre);    // uniform across the CTA
    if (cp && s_pref_cls != s_pre.cls) {           // 160 B, only when the class changes
      const uint32_t* src = reinterpret_cast<const uint32_t*>(cp);
      uint32_t* dst = reinterpret_cast<uint32_t*>(&s_pref);
      for (uint32_t i = threadIdx.x; i < sizeof(ClassPref) / 4; i += EVICT_THREADS) dst[i] = src[i];
      __syncthreads();
      if (threadIdx.x == 0) s_pref_cls = s_pre.cls;
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
    const ClassPref* scp = cp ? &s_pref : nullptr;
    const uint32_t pmax = s_pmax;
    for (uint32_t n = blockIdx.x * EVICT_THREADS + threadIdx.x; n < S.N; n += nw * EVICT_THREADS) {
      const uint64_t k = evict_node_key(S, E, s_pre, s_cls, scp, pmax, n, &err);
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
__global__ void evict_scan_kernel(const __grid_constant__ DevSession S, const __grid_constant__ EvictDev E) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < S.J) evict_scan_job(S, E, j);
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
  if (S.J) evict_scan_kernel<<<(S.J + 255) / 256, 256, 0, stream>>>(S, E);
  DevSession s = S; EvictDev ev = E;
  void* args[] = {(void*)&s, (void*)&ev};
  const void* fn = preempt ? (const void*)evict_kernel<1> : (const void*)evict_kernel<0>;
  return cudaLaunchCooperativeKernel(fn, dim3(workers + 1), dim3(EVICT_THREADS), args, 0, stream);
}

}  // namespace kb
