// kb_pipe.cuh — the allocate cycle as ONE persistent cooperative kernel (sm_90a).
//
// cycle_kernel<R, W>   grid = pipe_S scanner CTAs + 1 replayer CTA, all co-resident, one launch per kb_allocate.
//
//   scanner CTA   keeps pipe_tpc node tiles (TMA bulk copy at start) RESIDENT in shared memory for the whole cycle.
//                 Three warp groups (4 warps = 128 threads = one node per thread per tile) serve scan requests
//                 seq = g, g+3, ... concurrently: K1 predicate bitmask + K2 fused score (eval_pair) for the request's
//                 class over the CTA's nodes, warp bitonic top-32 (K3), group fold, list -> global; the LAST group to
//                 deliver (ticket) merges the pipe_S lists and publishes the request's top-32 (NCCL-LL style words:
//                 the payload carries its own sequence tag, no separate flag, no fence on the reader).
//                 Warp 12 (applier) follows the modification log and refreshes the resident tiles.
//   replayer CTA  warp 0 (main) walks the visits exactly like allocate.go:89-193: for the class of the next run it takes
//                 the look-ahead list that was requested a few visits earlier (stamp = log position at the request),
//                 PATCHES it — every node modified since the stamp is dropped from the list and re-evaluated from the
//                 replayer's own copy (hot ring) by the four patch warps — and replays: the prep teams (2 x 4 warps) have
//                 evaluated the list's candidates at placement depths 0..7 ahead of the visit (the state after k more
//                 placements of this class is a pure function of the record), so a step of the run is a warp arg-max plus
//                 a shared-memory read.  The writer warp writes modified records back, appends the log, publishes its
//                 head (st.release: no L1 invalidation on this SM) and, as the planner, owns the requested table: it posts
//                 the scan requests for the classes of the next visits from a PLAN command the main warp pushes per visit.
//                 The shadow warp pulls the job / queue rows of the next visits into L1.
//
// Exactness (same argument as the per-launch kernels, generalised to a stale list): let L be the exact top-32 of class c
// for the table state at log position s, floor = its 32nd key, M = nodes in log[s, now).  A node outside L and outside M
// is unmodified since s, so its current key is below floor.  Every node of M is re-evaluated on its current record.  The
// 32 best of (L \ M) U M are kept; the floor rises to the best key dropped.  A pick is certified iff best >= floor, else
// the run stops and a fresh list is requested (STOP_RESCAN).  A scanner may read a record WHILE it is being rewritten
// (torn read): that node is in log[s, now) for every list it can have influenced, so its entry is dropped and
// re-evaluated; a garbage key can only displace true candidates, which raises nothing above the published floor.
// tests/emu re-enacts the protocol (random staleness, garbage keys for in-flight nodes) against the oracle.
#pragma once

#include "kb_kernels.cuh"

namespace kb {

constexpr int PIPE_DEPTH = 8;              // placement depths a prep team evaluates per list entry (ahead of the visit)
constexpr int PIPE_PDEPTH = 4;             // ... and the patch warps per patch entry (on the visit's critical path: kept short;
                                           //     deeper states of a candidate come from the chain extension)
// 16 warps per CTA: four per scheduler (SM sub-partition, warp % 4), so ptxas may use 128 registers per thread (a 17th warp
// would put five on one scheduler: 96 registers and spills in the step loop).
// replayer CTA warp roles: the main warp (0) shares its scheduler only with patch warps (4, 8, 12), which run while it waits at
// their barrier or, as the pool builder, while it does a chain's bookkeeping; the prep teams, the writer / planner, the shadow prefetch and the fourth patch warp sit on the other three.
// scanner CTAs: PIPE_SCAN_GROUPS scan groups of 4 warps, then the applier warp.
constexpr int PIPE_PREP_TEAMS = 2, PIPE_PREP_TW = 4;
constexpr int PIPE_WARPS = 16;
constexpr int PIPE_THREADS = PIPE_WARPS * 32;
constexpr int PIPE_SCAN_GROUPS = 3;
constexpr int PIPE_W_APPLIER = 4 * PIPE_SCAN_GROUPS;
static_assert(PIPE_W_APPLIER < PIPE_WARPS, "scanner CTA: scan groups + applier");
enum PipeRole : int { ROLE_MAIN = 0, ROLE_PATCH = 1, ROLE_PREP = 2, ROLE_WRITER = 3, ROLE_SHADOW = 4, ROLE_NONE = 5 };
__device__ __forceinline__ void pipe_role(const int warp, int& role, int& idx) {
  idx = 0;
  if (warp == 0) { role = ROLE_MAIN; return; }
  if ((warp & 3) == 0) { role = ROLE_PATCH; idx = (warp >> 2) - 1; return; }                // 4, 8, 12 -> depth 0..2
  const int r = warp - 1 - (warp >> 2);                                                      // 1,2,3,5,6,7,9,10,11,13,14,15 -> 0..11
  if (r < PIPE_PREP_TEAMS * PIPE_PREP_TW) { role = ROLE_PREP; idx = r; return; }
  if (r == PIPE_PREP_TEAMS * PIPE_PREP_TW) { role = ROLE_WRITER; return; }
  if (r == PIPE_PREP_TEAMS * PIPE_PREP_TW + 1) { role = ROLE_SHADOW; return; }
  if (r == PIPE_PREP_TEAMS * PIPE_PREP_TW + 2) { role = ROLE_PATCH; idx = 3; return; }       // warp 15 -> depth 3
  role = ROLE_NONE;
}
static_assert(PIPE_PDEPTH == 4 && PIPE_PREP_TEAMS * PIPE_PREP_TW + 3 <= 12, "warp roles of the replayer CTA");
static_assert(PIPE_DEPTH % PIPE_PREP_TW == 0, "a prep warp owns depths w, w + TW, ...");
constexpr uint32_t PIPE_HOT = 128;         // hot ring: records of the most recent log entries (replayer shared memory)
constexpr uint32_t PIPE_RQ = 16;           // requested-table entries (most recent scan requests)
constexpr uint32_t PIPE_CMDS = 64;
constexpr long long PIPE_DEADLINE = 3000000000ll;     // cycles a wait may take before the cycle is aborted (error 3)

enum PipeCmd : uint32_t { PCMD_WB = 1, PCMD_PLAN = 2, PCMD_QUIT = 3 };
constexpr uint32_t PLAN_FORCE_BIT = 4u;      // PCMD_PLAN word: kind | PLAN_FORCE_BIT (request the next visit's class whatever the table holds) | job << 3

// ---- memory-model helpers ----
__device__ __forceinline__ uint32_t ld_relaxed_u32(const uint32_t* p) {
  uint32_t v; asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ uint32_t ld_acquire_u32(const uint32_t* p) {
  uint32_t v; asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ void st_release_u32(uint32_t* p, uint32_t v) {        // MEMBAR.ALL.GPU + store, no L1 invalidation
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void st_relaxed_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void ld_relaxed_2u64(const unsigned long long* p, unsigned long long& a, unsigned long long& b) {
  asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}
// progress word -> mapped host memory (debug builds of a session only; a store, so it never stalls the warp)
__device__ __forceinline__ void dbg_put(uint32_t* dbg, int i, uint32_t v) { if (dbg) *((volatile uint32_t*)(dbg + i)) = v; }
// Shared-memory mailboxes of the replayer CTA: ONE 8- or 16-byte word carries tag + payload, written / read by a single thread
// with a single access, so producer and consumer need no fence (a MEMBAR.SC.CTA on the main warp also waits for its
// outstanding global stores: hundreds of cycles per command).  Data a mailbox word announces (hot ring entries) was stored by
// the same warp before it; shared-memory accesses of one warp are performed in issue order.
__device__ __forceinline__ void sts_v4(void* p, uint32_t x, uint32_t y, uint32_t z, uint32_t w) {
  asm volatile("st.volatile.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"((uint32_t)__cvta_generic_to_shared(p)), "r"(x), "r"(y), "r"(z), "r"(w) : "memory");
}
__device__ __forceinline__ uint4 lds_v4(const void* p) {
  uint4 v;
  asm volatile("ld.volatile.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"((uint32_t)__cvta_generic_to_shared(p)) : "memory");
  return v;
}
__device__ __forceinline__ void sts_u64(void* p, unsigned long long v) {
  asm volatile("st.volatile.shared.u64 [%0], %1;" ::"r"((uint32_t)__cvta_generic_to_shared(p)), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long lds_u64(const void* p) {
  unsigned long long v;
  asm volatile("ld.volatile.shared.u64 %0, [%1];" : "=l"(v) : "r"((uint32_t)__cvta_generic_to_shared(p)) : "memory");
  return v;
}
__device__ __forceinline__ void compiler_fence() { asm volatile("" ::: "memory"); }
__device__ __forceinline__ void bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void bar_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }
// A bounded wait of the replayer CTA: poll done() until it holds (true), or until quit() holds or PIPE_DEADLINE cycles have passed
// (false; what that means is the caller's).  SLEEP: ns of __nanosleep between polls, 0 for a wait on the visit's critical path.
template <int SLEEP, typename Done, typename Quit>
__device__ __forceinline__ bool wait_until(Done done, Quit quit) {
  const long long deadline = clock64() + PIPE_DEADLINE;
  while (!done()) {
    if (quit() || clock64() > deadline) return false;
    if (SLEEP) __nanosleep(SLEEP);
  }
  return true;
}
template <int SLEEP, typename Done>
__device__ __forceinline__ bool wait_until(Done done) { return wait_until<SLEEP>(done, [] { return false; }); }

// record held in registers (column c at r[c]); NC = tile_ncols(R, W) is a compile-time constant here
struct RegAcc {
  const uint64_t* r; uint32_t R, W;
  __device__ __forceinline__ uint64_t col(uint32_t c) const { return r[c]; }
  __device__ __forceinline__ double idle(uint32_t k) const { return u64_as_double(col(col_idle(R, k))); }
  __device__ __forceinline__ double rel(uint32_t k) const { return u64_as_double(col(col_rel(R, k))); }
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

// NodeInfo.AddTask of one task of class c on a record (node_info.go:172-212 as allocate.go:160-183 drives it): Allocate
// consumes Idle when InitResreq <= Idle, else Pipeline consumes Releasing.  Returns that fits-idle bit of the state BEFORE.
// Branch-free selects: no dynamic register indexing.
template <int RR, int WW>
__device__ __forceinline__ bool advance_rec(uint64_t* rec, const ClassRec& c) {
  constexpr uint32_t R = RR, W = WW;
  RegAcc a{rec, R, W};
  const bool fi = res_less_equal(R, [&](uint32_t k) { return c.initreq[k]; }, [&](uint32_t k) { return a.idle(k); });
#pragma unroll
  for (uint32_t k = 0; k < R; ++k) {
    const double id = u64_as_double(rec[col_idle(R, k)]), rl = u64_as_double(rec[col_rel(R, k)]);
    rec[col_idle(R, k)] = double_as_u64(fi ? KB_DSUB(id, c.resreq[k]) : id);
    rec[col_rel(R, k)] = double_as_u64(fi ? rl : KB_DSUB(rl, c.resreq[k]));
  }
  rec[col_nz_cpu(R)] = (uint64_t)((int64_t)rec[col_nz_cpu(R)] + c.nz_cpu);
  rec[col_nz_mem(R)] = (uint64_t)((int64_t)rec[col_nz_mem(R)] + c.nz_mem);
  rec[col_pods(R)] = rec[col_pods(R)] + 1ull;
#pragma unroll
  for (uint32_t w = 0; w < W; ++w) rec[col_ports(R, W, w)] |= c.port_own[w] | (fi ? c.aff_own[w] : 0ull);      // aff_own: ClassRec
  return fi;
}

// bitonic sort / merge networks carrying a 32-bit payload with the key (descending, lane 0 = best)
__device__ __forceinline__ void warp_sort_desc_kv(uint64_t& v, uint32_t& pl, int lane) {
#pragma unroll
  for (int k = 2; k <= 32; k <<= 1) {
#pragma unroll
    for (int j = k >> 1; j > 0; j >>= 1) {
      const uint64_t o = __shfl_xor_sync(FULL, v, j);
      const uint32_t op = __shfl_xor_sync(FULL, pl, j);
      const bool take_max = (((lane & k) == 0) == ((lane & j) == 0));
      const bool take_o = take_max ? (o > v) : (o < v);
      v = take_o ? o : v; pl = take_o ? op : pl;
    }
  }
}
// top-32 of two descending lists with payloads; `dropped` = the best key that did not make it (0 if none)
__device__ __forceinline__ void warp_merge_top32_kv(uint64_t& a, uint32_t& ap, uint64_t b, uint32_t bp, uint64_t& dropped, int lane) {
  const uint64_t br = __shfl_sync(FULL, b, 31 - lane);
  const uint32_t bpr = __shfl_sync(FULL, bp, 31 - lane);
  const bool tb = br > a;
  const uint64_t lo = tb ? a : br;
  uint64_t v = tb ? br : a;
  uint32_t pl = tb ? bpr : ap;
  dropped = warp_max_u64(lo);
#pragma unroll
  for (int j = 16; j > 0; j >>= 1) {
    const uint64_t o = __shfl_xor_sync(FULL, v, j);
    const uint32_t op = __shfl_xor_sync(FULL, pl, j);
    const bool take_max = (lane & j) == 0;
    const bool take_o = take_max ? (o > v) : (o < v);
    v = take_o ? o : v; pl = take_o ? op : pl;
  }
  a = v; ap = pl;
}

// ---------------------------------------------------------------------------------------------
// scanner CTA
// ---------------------------------------------------------------------------------------------
struct ScanGroup {
  ClassRec cls;
  ClassPref pref;                        // preferred node-affinity terms of the class (a12), n == 0: none
  uint32_t cls_id, stamp, quit, is_last;
  uint32_t pmax, pnmax, wmax[4], wn[4];  // pass 1: max count over the feasible nodes, nodes reaching it
  uint64_t wl[4][KTOP];
};
struct ScanSmem {
  uint32_t applied;          // log entries applied to the resident tiles (volatile)
  uint32_t pad[3];
  uint64_t mbar;
  uint64_t pad2;
  ScanGroup grp[PIPE_SCAN_GROUPS];
};
__host__ __device__ constexpr size_t pipe_scan_header() { return ((sizeof(ScanSmem) + 127) / 128) * 128; }

template <int RR, int WW, int PREF>
__device__ __forceinline__ void pipe_scanner(const DevSession& S, unsigned char* smem_raw) {
  constexpr uint32_t R = RR, W = WW, NC = 2 * RR + 6 + 3 * WW;
  ScanSmem& sm = *reinterpret_cast<ScanSmem*>(smem_raw);
  uint64_t* tiles = reinterpret_cast<uint64_t*>(smem_raw + pipe_scan_header());
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  PipeG* pg = S.pg;
  const uint32_t cta = blockIdx.x, nS = S.pipe_S, tpc = S.pipe_tpc;
  const uint32_t t0 = cta * tpc, t1 = min(S.NT, t0 + tpc), ntl = t1 > t0 ? t1 - t0 : 0;
  constexpr uint32_t tile_u64 = NC * TILE_NODES;
  if (tid == 0) {
    sm.applied = 0;
    mbar_init(&sm.mbar, 1); fence_mbar_init();
    mbar_expect_tx(&sm.mbar, ntl * tile_u64 * 8u);
    for (uint32_t i = 0; i < ntl; ++i) tma_load_1d(tiles + (size_t)i * tile_u64, S.tiles + (size_t)(t0 + i) * tile_u64, tile_u64 * 8u, &sm.mbar);
  }
  __syncthreads();
  mbar_wait(&sm.mbar, 0);

  if (warp > PIPE_W_APPLIER) return;
  if (warp == PIPE_W_APPLIER) {
    // ---------------- applier: follow the modification log, refresh the resident copies of MY nodes ----------------
    uint32_t cursor = 0;
    for (;;) {
      const uint32_t head = ld_acquire_u32(&pg->log_head);
      if (head != cursor) {
        for (uint32_t base = cursor; base < head; base += 32) {
          const uint32_t i = base + lane;
          if (i < head) {
            const uint32_t node = __ldcg(&S.modlog[i]);
            const uint32_t t = node / TILE_NODES;
            if (t >= t0 && t < t1) {
              const uint64_t* g = S.tiles + (size_t)t * tile_u64 + (node % TILE_NODES);
              uint64_t* d = tiles + (size_t)(t - t0) * tile_u64 + (node % TILE_NODES);
              uint64_t tmp[NC];
#pragma unroll
              for (uint32_t c = 0; c < NC; ++c) tmp[c] = __ldcg(g + (size_t)c * TILE_NODES);
#pragma unroll
              for (uint32_t c = 0; c < NC; ++c) d[(size_t)c * TILE_NODES] = tmp[c];
            }
          }
        }
        __syncwarp();
        __threadfence_block();
        if (lane == 0) *((volatile uint32_t*)&sm.applied) = head;
        cursor = head;
      } else {
        if (ld_relaxed_u32(&pg->quit)) return;
        __nanosleep(64);
      }
    }
  }

  // ---------------- scan groups ----------------
  const int g = warp >> 2, wg = warp & 3, gt = tid & 127;
  ScanGroup& G = sm.grp[g];
  const int bar_id = 1 + g;
  for (uint32_t seq = (uint32_t)g;; seq += PIPE_SCAN_GROUPS) {
    const uint32_t slot = seq % PIPE_RING, tag = seq + 1;
    if (wg == 0) {
      unsigned long long w0 = 0, w1 = 0;
      uint32_t quit = 0;
      const long long deadline = clock64() + PIPE_DEADLINE;
      for (;;) {
        ld_relaxed_2u64(&pg->req[slot][0], w0, w1);
        if ((uint32_t)(w0 >> 32) == tag && (uint32_t)(w1 >> 32) == tag) break;
        if (ld_relaxed_u32(&pg->quit)) { quit = 1; break; }
        if (clock64() > deadline) { quit = 1; if (lane == 0) { pg->error = 3; st_release_u32(&pg->quit, 1u); } break; }
        __nanosleep(32);
      }
      if (lane == 0) { G.cls_id = (uint32_t)w0; G.stamp = (uint32_t)w1; G.quit = quit; }
    }
    bar_sync(bar_id, 128);
    if (G.quit) return;
    if (cta == 0 && gt == 0) dbg_put(S.dbg, 24 + g, (seq << 4) | 1u);
    const uint32_t cls_id = G.cls_id, stamp = G.stamp;
    {
      const uint32_t* src = reinterpret_cast<const uint32_t*>(&S.classes[cls_id]);
      uint32_t* dst = reinterpret_cast<uint32_t*>(&G.cls);
      for (uint32_t i = gt; i < sizeof(ClassRec) / 4; i += 128) dst[i] = src[i];
      if (PREF && S.class_pref) {
        const uint32_t* ps = reinterpret_cast<const uint32_t*>(&S.class_pref[cls_id]);
        uint32_t* pd = reinterpret_cast<uint32_t*>(&G.pref);
        for (uint32_t i = gt; i < sizeof(ClassPref) / 4; i += 128) pd[i] = ps[i];
      } else if (gt == 0) G.pref.n = 0;
    }
    {
      // the resident tiles must reflect every log entry below the request's stamp (entries at or above it are the replayer's patch)
      const long long deadline = clock64() + PIPE_DEADLINE;
      while (*((volatile uint32_t*)&sm.applied) < stamp) {
        if (clock64() > deadline) { pg->error = 3; st_release_u32(&pg->quit, 1u); break; }
        __nanosleep(32);
      }
      __threadfence_block();
    }
    bar_sync(bar_id, 128);
    // NodeAffinityPriority (a12): NormalizeReduce needs the max count over the FEASIBLE nodes of the whole table before a
    // single key can be built -> pass 1 over the resident tiles, one exchange between the scanner CTAs, then the keys
    const bool is_pref = PREF && S.cf.nodeorder && G.pref.n != 0;
    int64_t pmax = 0;
    if (is_pref) {
      uint32_t mymax = 0, myn = 0;
      for (uint32_t i = 0; i < ntl; ++i) {
        const uint32_t node = (t0 + i) * TILE_NODES + gt;
        if (node >= S.N) continue;
        ColAcc acc{tiles + (size_t)i * tile_u64, (uint32_t)gt, TILE_NODES, R, W};
        if (!eval_pair<RR, WW>(S.cf, G.cls, acc, node, nullptr)) continue;
        const uint32_t cnt = (uint32_t)pref_count(G.pref, acc, W);
        if (cnt > mymax) { mymax = cnt; myn = 1; } else if (cnt == mymax) myn += 1;
      }
      const uint32_t wm = __reduce_max_sync(FULL, mymax);
      const uint32_t wnn = __reduce_add_sync(FULL, mymax == wm ? myn : 0u);
      if (lane == 0) { G.wmax[wg] = wm; G.wn[wg] = wnn; }
      bar_sync(bar_id, 128);
      if (wg == 0) {
        uint32_t gm = 0, gn = 0;
#pragma unroll
        for (int w = 0; w < 4; ++w) { if (G.wmax[w] > gm) { gm = G.wmax[w]; gn = G.wn[w]; } else if (G.wmax[w] == gm) gn += G.wn[w]; }
        if (lane == 0) {
          st_relaxed_u64(&S.ppref[(size_t)slot * nS + cta], ((unsigned long long)gm << 32) | gn);
          __threadfence();
          atomicAdd(&pg->ticket_pref[slot], 1u);
        }
        const long long deadline = clock64() + PIPE_DEADLINE;
        while (ld_acquire_u32(&pg->ticket_pref[slot]) < nS) {
          if (clock64() > deadline) { pg->error = 3; st_release_u32(&pg->quit, 1u); break; }
          __nanosleep(32);
        }
        uint32_t am = 0, an = 0;
        for (uint32_t c2 = (uint32_t)lane; c2 < nS; c2 += 32) {
          const unsigned long long v = __ldcg(&S.ppref[(size_t)slot * nS + c2]);
          const uint32_t m2 = (uint32_t)(v >> 32), n2 = (uint32_t)v;
          if (m2 > am) { am = m2; an = n2; } else if (m2 == am) an += n2;
        }
        const uint32_t tm = __reduce_max_sync(FULL, am);
        const uint32_t tn = __reduce_add_sync(FULL, am == tm ? an : 0u);
        if (lane == 0) { G.pmax = tm; G.pnmax = tn; }
      }
      bar_sync(bar_id, 128);
      pmax = (int64_t)G.pmax;
    }
    uint64_t mylist = 0;
    for (uint32_t i = 0; i < ntl; ++i) {
      const uint32_t node = (t0 + i) * TILE_NODES + gt;
      uint64_t key = 0;
      if (node < S.N) {
        ColAcc acc{tiles + (size_t)i * tile_u64, (uint32_t)gt, TILE_NODES, R, W};
        key = eval_pair<RR, WW>(S.cf, G.cls, acc, node, nullptr);
        if (is_pref && key) key = add_pref_term(key, (int64_t)S.w_nodeaff, (int64_t)pref_count(G.pref, acc, W), pmax);
      }
      const uint64_t thr = __shfl_sync(FULL, mylist, 31);
      if (__any_sync(FULL, key > thr)) {
        key = warp_sort_desc(key, lane);
        mylist = warp_merge_top32(mylist, key, lane);
      }
    }
    if (wg) G.wl[wg][lane] = mylist;
    bar_sync(bar_id, 128);
    if (wg == 0) {
#pragma unroll
      for (int w = 1; w < 4; ++w) mylist = warp_merge_top32(mylist, G.wl[w][lane], lane);
      S.pcand[((size_t)slot * nS + cta) * KTOP + lane] = mylist;
      __threadfence();
      __syncwarp();
      if (lane == 0) {
        const uint32_t old = atomicAdd(&pg->ticket[slot], 1u);
        G.is_last = (old == nS - 1) ? 1u : 0u;
      }
    }
    bar_sync(bar_id, 128);
    if (G.is_last) {
      // ---------------- last group for this request: merge the CTAs' lists, publish ----------------
      __threadfence();
      uint64_t acc = 0;
      for (uint32_t c = (uint32_t)wg; c < nS; c += 4) {
        const uint64_t cur = __ldcg(&S.pcand[((size_t)slot * nS + c) * KTOP + lane]);
        const uint64_t thr = __shfl_sync(FULL, acc, 31);
        const uint64_t head = __shfl_sync(FULL, cur, 0);
        if (head > thr) acc = warp_merge_top32(acc, cur, lane);
      }
      if (wg) G.wl[wg][lane] = acc;
      bar_sync(bar_id, 128);
      if (wg == 0) {
#pragma unroll
        for (int w = 1; w < 4; ++w) acc = warp_merge_top32(acc, G.wl[w][lane], lane);
        if (lane == 0) {
          pg->ticket[slot] = 0;
          if (is_pref) {      // every CTA has left pass 1 (it delivered its list): the slot's pass-1 counter can be recycled
            pg->ticket_pref[slot] = 0;
            st_relaxed_u64(&pg->pref[slot][0], ((unsigned long long)tag << 32) | G.pmax);
            st_relaxed_u64(&pg->pref[slot][1], ((unsigned long long)tag << 32) | G.pnmax);
          }
        }
        __threadfence();
        st_relaxed_u64(&pg->list[slot][2 * lane], ((unsigned long long)tag << 32) | (acc & 0xFFFFFFFFull));
        st_relaxed_u64(&pg->list[slot][2 * lane + 1], ((unsigned long long)tag << 32) | (acc >> 32));
      }
      bar_sync(bar_id, 128);      // G.wl / G.is_last are reused by the next request
    }
  }
}

// ---------------------------------------------------------------------------------------------
// replayer CTA
// ---------------------------------------------------------------------------------------------
// One prepared look-ahead list: everything the replay needs about the request's 32 candidates, evaluated AHEAD of the visit
// by a prep team (list wait, record gather and the depth chain are off the replay's critical path).  Valid for every entry
// whose node is not in log[stamp, now): such a node is unmodified since the stamp, so its record — read at any time after
// the stamp — and every key derived from it are current.  Entries of modified nodes are dropped at the visit (the patch
// entry of the node speaks for it).
template <int NC>
struct PrepBuf {
  ClassRec cls;
  uint64_t list[KTOP];                         // the request's list as published (descending, 0-padded); [31] = floor
  uint64_t key[PIPE_DEPTH][KTOP];              // key of entry l after d more placements of the class
  uint32_t fi[PIPE_DEPTH];                     // fits-idle ballots of the same states
  uint64_t rec[NC][KTOP];                      // entry l's record (state at depth 0)
  // NodeAffinityPriority (a12): the class's preferred terms, the request's normalisation (max count over the feasible
  // nodes at the stamp, nodes reaching it) and entry l's own count.  Lists of such classes are only used fresh.
  ClassPref pref;
  uint32_t is_pref, pmax, pnmax, pad_pref;
  int32_t cnt[KTOP];
};

template <int NC>
struct ReplaySmem {
  Ctl ctl;
  // visit descriptor (main warp -> patch warps)
  uint32_t v_pb, v_stamp, v_npatch, v_pvalid, v_quit, v_err, v_count;
  uint32_t v_buf;                              // pkey / pfi buffer of the pool being replayed (main warp; the patch warps fill it)
  long long t_cycle0;                          // main warp: clock64 at the first visit (kept here, not in a register)
  uint32_t v_mode;                             // at the go barrier: 0 patch the visit's list, 1 build the next chain's pool (b_*)
  uint32_t pnode[32];                          // patch entry i: node of log entry v_stamp + i (valid bit in v_pvalid: latest entry of its node)
  // patch entry i after d more placements; two buffers: the builder fills one while the running chain still reads the other
  uint64_t pkey[2][PIPE_PDEPTH][KTOP];
  uint32_t pfi[2][PIPE_PDEPTH];
  // pool builder (the patch warps in mode 1): the pool of the next visit chain, built while the main warp finishes this one.
  // Descriptor (main -> builder, written before the go barrier): predicted class, class of this chain, log head after this
  // chain's append, this chain's prepared list (slot of pb, its stamp), pkey buffer to fill, and per main-warp lane its
  // candidate's node and slot | placements << 8 (0 placements: unmodified).
  uint32_t b_gen, b_cls, b_ccls, b_head, b_pb, b_stamp, b_buf;
  uint32_t b_mnode[32], b_mslot[32];
  uint32_t b_plan;                             // volatile: command index of this chain's PCMD_PLAN once pushed (0 = not yet)
  uint32_t b_abort;                            // volatile: the main warp will not take this pool
  uint32_t b_ring, b_done;                     // volatile: b_gen once the hot ring holds this chain's records / once the build ended
  uint32_t b_ok, b_seq, b_lstamp, b_npatch, b_pvalid;   // result: pool built from prepared list b_seq (stamp b_lstamp)
  uint32_t b_urgent, b_waited;                 // result: no usable list at the first look / the prepared list was not ready yet
  uint64_t b_key[KTOP]; uint32_t b_slot[KTOP]; uint64_t b_floor;
  uint32_t in_use2;                            // seq + 1 of the prepared list the builder holds (volatile; second word of `claim`)
  uint64_t cmp_key[KTOP]; uint32_t cmp_slot[KTOP];       // compaction scratch of the main warp
  uint32_t step_rec[32];                       // a run's steps not yet written out: owner lane | fits-idle << 5
  uint64_t psort_key[KTOP]; uint32_t psort_slot[KTOP];   // patch entries' fresh keys, sorted (descending); slot = 32 + i
  // chain extension of ONE pool slot beyond PIPE_DEPTH
  uint64_t ext_key[32]; uint32_t ext_fi, ext_slot, ext_base, ext_pad;
  // hot ring: entry i of the modification log lives at i % PIPE_HOT until the writer has written it back and no list needs it
  uint32_t hot_node[PIPE_HOT], hot_cnt[PIPE_HOT], hot_cls[PIPE_HOT];
  uint64_t hot_rec[NC][PIPE_HOT];
  // requested table (request seq lives at seq % PIPE_RQ, and so does its prepared list)
  // {class, seq + 1 (0 = empty), stamp, 0}: one 16-byte word per entry, written by the planner (writer warp), read by main
  uint4 rq_ent[PIPE_RQ];
  uint32_t in_use;                             // seq + 1 of the prepared list the main warp is replaying (volatile: main -> planner)
  uint32_t posting;                            // seq + 1 of the request the planner is entering (volatile: planner -> main)
  uint32_t n_requests;                         // planner -> main at PCMD_QUIT
  unsigned long long rq_word[PIPE_RQ];         // (seq + 1) << 32 | class: request seq exists (one word, main -> prep teams)
  uint32_t pb_ready[PIPE_RQ];                  // seq + 1 once pb[seq % PIPE_RQ] holds request seq (volatile: prep -> main)
  uint32_t prep_done[PIPE_PREP_TEAMS];         // requests a team has finished (its next seq; volatile)
  uint32_t prep_status[PIPE_PREP_TEAMS];       // warp 0 of a team -> its other warps
  // main -> writer command ring
  uint4 cmd[PIPE_CMDS];                        // {index + 1, kind, a, b}: one 16-byte word per command
  uint32_t cmd_tail;                           // commands the writer has finished (volatile)
  uint32_t pub_head;                           // log entries the writer has published (volatile)
  uint32_t sink;
  PrepBuf<NC> pb[PIPE_RQ];
};

// newest request for class `cls` in the requested table (whole warp): found; seq / stamp by reference
template <int NC>
__device__ __forceinline__ bool rq_find(const ReplaySmem<NC>& sm, const int lane, const uint32_t cls, uint32_t& seq, uint32_t& stamp) {
  uint4 e = make_uint4(0u, 0u, 0u, 0u);
  if (lane < (int)PIPE_RQ) e = lds_v4(&sm.rq_ent[lane]);
  const bool m = e.y != 0u && e.x == cls;
  const uint32_t s1 = m ? e.y : 0u;
  const uint32_t best = __reduce_max_sync(FULL, s1);
  if (best == 0) return false;
  const int src = __ffs(__ballot_sync(FULL, m && s1 == best)) - 1;
  seq = best - 1u;
  stamp = __shfl_sync(FULL, e.z, src);
  return true;
}

// a class with preferred node-affinity terms: its keys are normalised by the max count over the nodes feasible AT THE STAMP, so
// only a list of the current table state will do (the replay then tracks the feasible max-count nodes itself)
template <int PREF>
__device__ __forceinline__ bool pref_class(const DevSession& S, const uint32_t cls) {
  return PREF && S.class_pref != nullptr && S.cf.nodeorder && S.class_pref[cls].n != 0;
}
// may a list stamped at `stamp` serve a visit that starts at log position `head`: at most age_max entries behind, requested at or
// after fresh_floor (after a rescan stop), and for a class with preferred terms (pref) of the current table state
__device__ __forceinline__ bool list_usable(const uint32_t head, const uint32_t stamp, const uint32_t age_max, const uint32_t fresh_floor, const bool pref) {
  return (head - stamp) <= age_max && stamp >= fresh_floor && (!pref || stamp == head);
}

// Claim prepared list `seq` against the planner recycling its buffer (whole warp): `word` is in_use (the main warp's visit) or
// in_use2 (the pool builder).  One side of the handshake with `post` in the writer warp: store the word, fence, then read posting
// and the table entry.  false: the planner is recycling the buffer, the word is cleared again.
template <int NC>
__device__ __forceinline__ bool claim(ReplaySmem<NC>& sm, uint32_t* word, const uint32_t seq, const int lane) {
  uint32_t ok = 1;
  if (lane == 0) {
    *((volatile uint32_t*)word) = seq + 1;
    __threadfence_block();
    const uint32_t po = *((volatile uint32_t*)&sm.posting);
    const uint4 e = lds_v4(&sm.rq_ent[seq % PIPE_RQ]);
    if (po == seq + 1 + PIPE_RQ || e.y != seq + 1) { *((volatile uint32_t*)word) = 0; ok = 0; }
  }
  return __shfl_sync(FULL, ok, 0) != 0;
}

// Patch set of a list stamped at `stamp`: log entries [stamp, stamp + npatch), entry i in lane i.  pn: its node (lanes from npatch
// on hold distinct fillers); returns whether it is the latest entry of its node, the only one that holds the node's current record.
template <int NC>
__device__ __forceinline__ bool patch_set(const ReplaySmem<NC>& sm, const uint32_t stamp, const uint32_t npatch, uint32_t& pn, const int lane) {
  pn = 0xFFFFFFF0u - (uint32_t)lane;
  const bool pv = (uint32_t)lane < npatch;
  if (pv) pn = sm.hot_node[(stamp + lane) % PIPE_HOT];
  const unsigned same = __match_any_sync(FULL, pn);
  return pv && (same >> (lane + 1)) == 0u;
}

// record (state at depth 0) of pool slot `slot` of a pool built from prepared list P and the patch set at `stamp`: list entry
// slot < 32 from the prepared buffer, patch entry slot - 32 from the hot ring
template <int NC>
__device__ __forceinline__ void pool_rec(const ReplaySmem<NC>& sm, const PrepBuf<NC>& P, const uint32_t stamp, const uint32_t slot, uint64_t* r) {
  const uint32_t l = slot & 31u;
  if ((slot >> 5) == 0) {
#pragma unroll
    for (uint32_t cc = 0; cc < NC; ++cc) r[cc] = P.rec[cc][l];
  } else {
    const uint32_t hi = (stamp + l) % PIPE_HOT;
#pragma unroll
    for (uint32_t cc = 0; cc < NC; ++cc) r[cc] = sm.hot_rec[cc][hi];
  }
}

// Ring append at the end of a visit chain: each candidate with placements (depth > 0; pool slot `slot`, node `node`) -> its state
// after them into the hot ring, in lane order, as the log entries that end at `head`.  First waits until the writer has written
// back the ring entries this overwrites; false: that wait timed out (the records are still written).
template <int RR, int WW>
__device__ __forceinline__ bool ring_append(ReplaySmem<2 * RR + 6 + 3 * WW>& sm, const PrepBuf<2 * RR + 6 + 3 * WW>& P, const uint32_t stamp,
                                            const uint32_t head, const uint32_t slot, const uint32_t depth, const uint32_t node,
                                            const uint32_t cls_id, const int lane) {
  constexpr uint32_t NC = 2 * RR + 6 + 3 * WW;
  const unsigned mm = __ballot_sync(FULL, depth > 0);
  const bool in_time = wait_until<20>([&] { return head - *((volatile uint32_t*)&sm.pub_head) <= PIPE_HOT - PIPE_PATCH; });
  if (depth > 0) {
    uint64_t r[NC];
    pool_rec(sm, P, stamp, slot, r);
    for (uint32_t k = 0; k < depth; ++k) advance_rec<RR, WW>(r, P.cls);
    const uint32_t base = head - (uint32_t)__popc(mm);
    const uint32_t hi = (base + (uint32_t)__popc(mm & ((1u << lane) - 1u))) % PIPE_HOT;
#pragma unroll
    for (uint32_t cc = 0; cc < NC; ++cc) sm.hot_rec[cc][hi] = r[cc];
    sm.hot_node[hi] = node; sm.hot_cnt[hi] = depth; sm.hot_cls[hi] = cls_id;
  }
  return in_time;
}

// Patch entry `lane` of the log window [stamp, stamp + npatch) evaluated at placement depth d for class `cls` (valid: the latest
// entry of its node) -> pkey[buf][d] / pfi[buf][d]; depth 0 also leaves the entries sorted in psort_*.
template <int RR, int WW>
__device__ __forceinline__ void patch_eval(const DevSession& S, ReplaySmem<2 * RR + 6 + 3 * WW>& sm, const ClassRec& cls, const uint32_t stamp,
                                           const uint32_t npatch, const bool have, const uint32_t node, const uint32_t buf, const int d, const int lane) {
  constexpr uint32_t R = RR, W = WW, NC = 2 * RR + 6 + 3 * WW;
  uint64_t key = 0;
  bool fi = false;
  if (have) {
    uint64_t rec[NC];
    const uint32_t hi = (stamp + (uint32_t)lane) % PIPE_HOT;
#pragma unroll
    for (uint32_t c = 0; c < NC; ++c) rec[c] = sm.hot_rec[c][hi];
    for (int k = 0; k < d; ++k) advance_rec<RR, WW>(rec, cls);
    RegAcc acc{rec, R, W};
    key = eval_pair<RR, WW>(S.cf, cls, acc, node, &fi);
  }
  sm.pkey[buf][d][lane] = key;
  const unsigned fim = __ballot_sync(FULL, have && fi);
  if (lane == 0) sm.pfi[buf][d] = fim;
  if (d == 0) {
    // sorted (descending) for the merge with the list: rank = keys greater than mine (+ equal ones — only zeros — of lower
    // lanes), read from shared memory with broadcast loads: ~4x shorter than a 15-stage shuffle network on this critical path.
    // Lanes from npatch on hold zeros and rank behind every valid entry, in lane order.
    __syncwarp();
    uint32_t rank = (uint32_t)lane;
    if ((uint32_t)lane < npatch) {
      rank = 0;
      for (uint32_t l2 = 0; l2 < npatch; ++l2) {
        const uint64_t o = sm.pkey[buf][0][l2];
        rank += (o > key || (o == key && l2 < (uint32_t)lane)) ? 1u : 0u;
      }
    }
    sm.psort_key[rank] = key; sm.psort_slot[rank] = 32u + (uint32_t)lane;
  }
}

// the prepared list minus the nodes of the patch set (pn: lane i holds patch entry i's node, npatch of them), compacted in list
// order: lane-owned candidates (key at depth 0, slot = list entry).  `scratch` is the calling warp's own.
__device__ __forceinline__ void list_minus_patch(const uint64_t* list, const uint64_t* key0, const uint32_t pn, const uint32_t npatch,
                                                 uint64_t* scratch_key, uint32_t* scratch_slot, uint64_t& cur_key, uint32_t& slot, const int lane) {
  const uint64_t lk = list[lane];
  const uint32_t lnode = key_node(lk);
  bool ok = lk != 0;
  for (uint32_t i = 0; i < npatch; ++i) { const uint32_t o = __shfl_sync(FULL, pn, (int)i); ok = ok & (o != lnode); }   // no short-circuit: every lane takes part in the shuffle
  const uint64_t k0 = ok ? key0[lane] : 0ull;
  const unsigned am = __ballot_sync(FULL, k0 != 0);
  if (k0) { const uint32_t rank = (uint32_t)__popc(am & ((1u << lane) - 1u)); scratch_key[rank] = k0; scratch_slot[rank] = (uint32_t)lane; }
  __syncwarp();
  const bool in = (uint32_t)lane < (uint32_t)__popc(am);
  cur_key = in ? scratch_key[lane] : 0ull;
  slot = in ? scratch_slot[lane] : 0u;
  __syncwarp();
}

// The pool of a visit from prepared list P and its patch set (pn, npatch; see list_minus_patch): lane-owned candidates (cur_key,
// slot), the list's compacted entries merged with the patch entries' sorted depth-0 keys (psort_*, in place once wait_patch() has
// returned).  Returns the floor: the list's 32nd key, or the best key the merge dropped if that is higher.
template <int NC, typename WaitPatch>
__device__ __forceinline__ uint64_t pool_complete(const ReplaySmem<NC>& sm, const PrepBuf<NC>& P, const uint32_t pn, const uint32_t npatch,
                                                  uint64_t* scratch_key, uint32_t* scratch_slot, uint64_t& cur_key, uint32_t& slot,
                                                  const int lane, WaitPatch wait_patch) {
  list_minus_patch(P.list, P.key[0], pn, npatch, scratch_key, scratch_slot, cur_key, slot, lane);
  const uint64_t f0 = P.list[KTOP - 1];
  uint64_t dropped = 0;
  if (npatch) {
    wait_patch();
    warp_merge_top32_kv(cur_key, slot, sm.psort_key[lane], sm.psort_slot[lane], dropped, lane);
  }
  return f0 > dropped ? f0 : dropped;
}

// Pool builder: the four patch warps prepare the pool of the NEXT visit chain while the main warp writes this chain's decisions,
// sums and control plane.  Depth-0 warp: this chain's modified candidates -> hot ring (ring_append: the records the write-back
// command publishes), a usable prepared list of the predicted class (pref_class, list_usable: the rule of the main warp and the
// planner), claimed with in_use2, then the pool (patch_set, pool_complete) the main warp would build at the visit start from the
// same list.  Every warp evaluates its depth of the patch set.  The main warp takes the pool only if the visit has the predicted
// class and starts at b_head.
template <int RR, int WW, int PREF>
__device__ __forceinline__ void pipe_build(const DevSession& S, ReplaySmem<2 * RR + 6 + 3 * WW>& sm, const int d, const int lane) {
  constexpr uint32_t NC = 2 * RR + 6 + 3 * WW;
  const uint32_t gen = sm.b_gen, cls_id = sm.b_cls, head = sm.b_head, buf = sm.b_buf;
  if (d == 0) {
    const uint32_t ms = sm.b_mslot[lane];
    if (!ring_append<RR, WW>(sm, sm.pb[sm.b_pb], sm.b_stamp, head, ms & 63u, ms >> 8, sm.b_mnode[lane], sm.b_ccls, lane))
      *((volatile uint32_t*)&sm.v_err) = 1;
    __syncwarp();
    __threadfence_block();
    if (lane == 0) *((volatile uint32_t*)&sm.b_ring) = gen;
    // ---- which list (fresh_floor is 0 after a chain that did not rescan) ----
    const bool pref = pref_class<PREF>(S, cls_id);
    auto off = [&] { return *((volatile uint32_t*)&sm.b_abort) || *((volatile uint32_t*)&sm.v_err); };    // dropped / the cycle failed
    uint32_t seq = 0, stamp = 0, ok = 0;
    if (lane == 0) { sm.b_urgent = 0; sm.b_waited = 0; }
    for (bool waited = false;;) {
      bool usable = rq_find<NC>(sm, lane, cls_id, seq, stamp);
      usable = usable && list_usable(head, stamp, PIPE_PATCH, 0u, pref);
      if (usable) { ok = claim(sm, &sm.in_use2, seq, lane) ? 1u : 0u; break; }
      if (waited) break;
      if (lane == 0) sm.b_urgent = 1;
      // the planner judges the table by the same rule at this chain's PCMD_PLAN: wait until it has, look once more
      uint32_t stop = 0;
      if (lane == 0) {
        stop = !wait_until<20>([&] {
          const uint32_t pl = *((volatile uint32_t*)&sm.b_plan);
          return pl && (int32_t)(*((volatile uint32_t*)&sm.cmd_tail) - pl) >= 0;
        }, off);
      }
      if (__shfl_sync(FULL, stop, 0)) break;
      waited = true;
    }
    if (ok) {
      // the prep team's buffer (the main warp's wait at a visit start)
      uint32_t stop = 0;
      if (lane == 0) {
        auto ready = [&] { return *((volatile uint32_t*)&sm.pb_ready[seq % PIPE_RQ]) == seq + 1; };
        if (!ready()) sm.b_waited = 1;
        stop = !wait_until<20>(ready, off) || *((volatile uint32_t*)&sm.b_abort);      // dropped meanwhile: no evaluation
      }
      if (__shfl_sync(FULL, stop, 0)) { ok = 0; if (lane == 0) *((volatile uint32_t*)&sm.in_use2) = 0; }
    }
    if (lane == 0) { sm.b_ok = ok; sm.b_seq = seq; sm.b_lstamp = stamp; }
    __threadfence_block();
  }
  bar_sync(4, PIPE_PDEPTH * 32);                 // the list (or none) is chosen
  if (sm.b_ok) {
    const uint32_t stamp = sm.b_lstamp, pbi = sm.b_seq % PIPE_RQ, npatch = head - stamp;
    const PrepBuf<NC>& P = sm.pb[pbi];
    compiler_fence();
    uint32_t pn;
    const bool latest = patch_set(sm, stamp, npatch, pn, lane);
    patch_eval<RR, WW>(S, sm, P.cls, stamp, npatch, latest, pn, buf, d, lane);
    if (d == 0) {
      uint64_t cur_key; uint32_t slot;
      const uint64_t floor_key = pool_complete(sm, P, pn, npatch, sm.b_key, sm.b_slot, cur_key, slot, lane, [] { __syncwarp(); });
      sm.b_key[lane] = cur_key; sm.b_slot[lane] = slot;
      const unsigned pvalid = __ballot_sync(FULL, latest);
      if (lane == 0) { sm.b_floor = floor_key; sm.b_npatch = npatch; sm.b_pvalid = pvalid; }
    }
    __threadfence_block();
  }
  bar_sync(4, PIPE_PDEPTH * 32);                 // every depth is in place
  if (d == 0 && lane == 0) *((volatile uint32_t*)&sm.b_done) = gen;
}

// patch warps (one per placement depth): patch entry `lane` = the current record of a node modified since the list's stamp,
// from the hot ring (shared memory) — the only evaluation left on the replay's critical path
template <int RR, int WW, int PREF>
__device__ __forceinline__ void pipe_patch_warp(const DevSession& S, ReplaySmem<2 * RR + 6 + 3 * WW>& sm, const int d, const int lane) {
  for (;;) {
    bar_sync(1, (1 + PIPE_PDEPTH) * 32);         // go
    if (*((volatile uint32_t*)&sm.v_quit)) return;
    if (sm.v_mode) { pipe_build<RR, WW, PREF>(S, sm, d, lane); continue; }       // the main warp does not wait for a build here
    const bool have = ((sm.v_pvalid >> lane) & 1u) != 0;
    patch_eval<RR, WW>(S, sm, sm.pb[sm.v_pb].cls, sm.v_stamp, sm.v_npatch, have, sm.pnode[lane], sm.v_buf, d, lane);
    bar_sync(1, (1 + PIPE_PDEPTH) * 32);         // done
  }
}

// prep team (PIPE_PREP_TW warps): requests seq = team, team + PIPE_PREP_TEAMS, ...  Waits for the scanners' answer, gathers the
// 32 records, evaluates the depth chain (warp w: depths w, w + TW, ...) and publishes pb[seq % PIPE_RQ].
template <int RR, int WW, int PREF>
__device__ __forceinline__ void pipe_prep_warp(const DevSession& S, ReplaySmem<2 * RR + 6 + 3 * WW>& sm, const int team, const int w, const int lane) {
  constexpr uint32_t R = RR, W = WW, NC = 2 * RR + 6 + 3 * WW;
  PipeG* pg = S.pg;
  const int bar_id = 2 + team;
  for (uint32_t seq = (uint32_t)team;; seq += PIPE_PREP_TEAMS) {
    const uint32_t idx = seq % PIPE_RQ, slot = seq % PIPE_RING, tag = seq + 1;
    PrepBuf<NC>& P = sm.pb[idx];
    if (w == 0) {
      // warp 0 of the team waits (for the request to exist, then for the scanners' answer) and decides for the team, so that
      // all four warps leave together when the cycle ends
      uint32_t status = 0;                      // 0 ok, 1 quit, 2 timeout (kept warp-uniform)
      uint32_t rcls = 0;
      if (lane == 0) {
        unsigned long long rw;
        while ((uint32_t)((rw = lds_u64(&sm.rq_word[idx])) >> 32) != tag) {
          if (*((volatile uint32_t*)&sm.v_quit)) { status = 1; break; }
          __nanosleep(40);
        }
        rcls = (uint32_t)rw;
      }
      status = __shfl_sync(FULL, status, 0);
      rcls = __shfl_sync(FULL, rcls, 0);
      unsigned long long w0 = 0, w1 = 0;
      if (status == 0) {
        const uint32_t* src = reinterpret_cast<const uint32_t*>(&S.classes[rcls]);
        uint32_t* dst = reinterpret_cast<uint32_t*>(&P.cls);
        for (uint32_t i = lane; i < sizeof(ClassRec) / 4; i += 32) dst[i] = __ldg(src + i);
        if (PREF && S.class_pref) {
          const uint32_t* ps = reinterpret_cast<const uint32_t*>(&S.class_pref[rcls]);
          uint32_t* pd = reinterpret_cast<uint32_t*>(&P.pref);
          for (uint32_t i = lane; i < sizeof(ClassPref) / 4; i += 32) pd[i] = __ldg(ps + i);
        } else if (lane == 0) P.pref.n = 0;
        // the request's list: lane l polls its own two LL words (payload + tag in one 8-byte word each)
        const long long deadline = clock64() + PIPE_DEADLINE;
        for (;;) {
          ld_relaxed_2u64(&pg->list[slot][2 * lane], w0, w1);
          const bool okl = (uint32_t)(w0 >> 32) == tag && (uint32_t)(w1 >> 32) == tag;
          if (__all_sync(FULL, okl)) break;
          const uint32_t st = *((volatile uint32_t*)&sm.v_quit) ? 1u : (clock64() > deadline ? 2u : 0u);
          status = __shfl_sync(FULL, st, 0);     // nobody waits for this list any more / timeout: lane 0 decides
          if (status) break;
          __nanosleep(20);
        }
      }
      P.list[lane] = status ? 0ull : ((w0 & 0xFFFFFFFFull) | (w1 << 32));
      __syncwarp();
      if (lane == 0) {
        const bool isp = PREF && !status && S.cf.nodeorder && P.pref.n != 0;
        P.is_pref = isp ? 1u : 0u; P.pmax = 0; P.pnmax = 0;
        if (isp) {          // written before the list words (fence in between): present once the list is
          unsigned long long a = 0, b = 0;
          if (!wait_until<0>([&] {
                ld_relaxed_2u64(&pg->pref[slot][0], a, b);
                return (uint32_t)(a >> 32) == tag && (uint32_t)(b >> 32) == tag;
              }))
            status = 2;
          P.pmax = (uint32_t)a; P.pnmax = (uint32_t)b;
        }
        sm.prep_status[team] = status; if (status == 2) sm.v_err = 1;
      }
      __threadfence_block();
    }
    if (w == 0 && lane == 0) dbg_put(S.dbg, 8 + team, (seq << 4) | 1u);
    bar_sync(bar_id, PIPE_PREP_TW * 32);        // P.cls, P.list and the team's status are in place
    if (*((volatile uint32_t*)&sm.prep_status[team]) == 1) return;
    const uint64_t listkey = P.list[lane];
    const uint32_t node = key_node(listkey);
    const bool have = listkey != 0 && node < S.N;
    uint64_t rec[NC];
#pragma unroll
    for (uint32_t c = 0; c < NC; ++c) rec[c] = 0;
    if (have) {
      const uint64_t* g = S.tiles + (size_t)(node / TILE_NODES) * ((size_t)NC * TILE_NODES) + (node % TILE_NODES);
#pragma unroll
      for (uint32_t c = 0; c < NC; ++c) rec[c] = __ldcg(g + (size_t)c * TILE_NODES);
    }
    const bool is_pref = PREF && P.is_pref != 0;
    int32_t pcnt = 0;
    if (is_pref && have) { RegAcc a0{rec, R, W}; pcnt = pref_count(P.pref, a0, W); }      // labels do not change with placements
    if (w == 0) {
#pragma unroll
      for (uint32_t c = 0; c < NC; ++c) P.rec[c][lane] = rec[c];
      P.cnt[lane] = pcnt;
    }
    for (int k = 0; k < w; ++k) advance_rec<RR, WW>(rec, P.cls);
#pragma unroll 1
    for (int d = w; d < PIPE_DEPTH; d += PIPE_PREP_TW) {
      uint64_t key = 0;
      bool fi = false;
      if (have) {
        RegAcc acc{rec, R, W};
        key = eval_pair<RR, WW>(S.cf, P.cls, acc, node, &fi);
        if (is_pref) key = add_pref_term(key, (int64_t)S.w_nodeaff, (int64_t)pcnt, (int64_t)P.pmax);
      }
      P.key[d][lane] = key;
      const unsigned fim = __ballot_sync(FULL, have && fi);
      if (lane == 0) P.fi[d] = fim;
      if (d + PIPE_PREP_TW < PIPE_DEPTH)
        for (int k = 0; k < PIPE_PREP_TW; ++k) advance_rec<RR, WW>(rec, P.cls);
    }
    __threadfence_block();
    if (lane == 0) dbg_put(S.dbg, 16 + team * 4 + w, (seq << 4) | 2u);
    bar_sync(bar_id, PIPE_PREP_TW * 32);        // every depth is in place
    if (w == 0 && lane == 0) {
      *((volatile uint32_t*)&sm.pb_ready[idx]) = tag;
      *((volatile uint32_t*)&sm.prep_done[team]) = seq + PIPE_PREP_TEAMS;
    }
  }
}

// shadow warp: pulls the job / queue rows the control plane will read at the next visits into this SM's L1 (the replayer CTA is
// the only writer of those tables, so its L1 stays coherent): the jobs at the head of the current queue's static order, their
// task order rows, the queue rows.  Read-only hints; nothing depends on what it reads.
template <int NC>
__device__ __forceinline__ void pipe_shadow_warp(const DevSession& S, ReplaySmem<NC>& sm, const int lane) {
  uint32_t seen = 0;
  uint32_t acc = 0;
  for (;;) {
    uint32_t v;
    while ((v = *((volatile uint32_t*)&sm.v_count)) == seen) {
      if (*((volatile uint32_t*)&sm.v_quit)) { if (lane == 0) sm.sink = acc; return; }
      __nanosleep(100);
    }
    seen = v;
    const uint32_t q = *((volatile uint32_t*)&sm.ctl.cur_queue);
    if (q >= S.Q) continue;
    const uint32_t R = S.cf.R;
    const uint32_t h = S.q_static_head[q], hend = S.q_static_off[q + 1];
    // lanes 0..7: one upcoming job each
    if (lane < 8 && h + (uint32_t)lane < hend) {
      const uint32_t jn = S.q_static[h + lane];
      const uint32_t pn = S.job_pos[jn], en = S.job_ord_off[jn + 1];
      acc += (uint32_t)S.job_ready[jn] + (uint32_t)S.job_min_avail[jn] + S.job_placed[jn] + S.job_queue[jn] + (uint32_t)S.job_prio[jn] + S.job_tb_rank[jn];
      acc += (uint32_t)double_as_u64(S.job_share[jn]);
      for (uint32_t k = 0; k < R; ++k) acc += (uint32_t)double_as_u64(S.job_alloc[(size_t)k * S.J + jn]);
      if (pn < en) {
        acc += S.ord_class[pn] + S.ord_run[pn] + S.ord_task[pn] + S.ord_task[min(en - 1, pn + 31)];
        acc += S.ord_chain[(size_t)pn * (KB_CHAIN_MAX - 1)] + S.ord_chain[(size_t)pn * (KB_CHAIN_MAX - 1) + KB_CHAIN_MAX - 2];
      }
    }
    if ((uint32_t)lane < R) acc += (uint32_t)double_as_u64(S.q_allocated[(size_t)lane * S.Q + q]) + (uint32_t)double_as_u64(S.q_deserved[(size_t)lane * S.Q + q]);
    acc += S.q_deserved_present[q] + (uint32_t)double_as_u64(S.q_share[q]);
    if (S.Q > 1) acc += prefetch_queue_heap<true>(S, *((volatile uint32_t*)&sm.ctl.qheap_len), lane);
  }
}

// writer / planner warp: write-backs, log, requests — everything that needs a membar, off the replay's critical path
template <int RR, int WW, int PREF>
__device__ __forceinline__ void pipe_writer_warp(const DevSession& S, ReplaySmem<2 * RR + 6 + 3 * WW>& sm, const int lane) {
  constexpr uint32_t R = RR, NC = 2 * RR + 6 + 3 * WW;
  PipeG* pg = S.pg;
  uint32_t tail = 0;
  uint32_t next_seq = 0;         // scan requests posted
  // Enter request next_seq for class `cls`: table entry, the prep team's word, the scanners' slot.  The prepared buffer and the
  // table entry of request seq - PIPE_RQ are recycled: its team must be through with it, and the main warp must not be replaying
  // it.  Both sides write their word, fence, then read the other's (main: in_use then posting + entry; here: posting then in_use),
  // so at least one of them sees the other and steps back; a request that steps back is simply not made (a later plan repeats it).
  auto post = [&](const uint32_t cls, const uint32_t head) {
    const uint32_t seq = next_seq;
    if (seq >= PIPE_RQ && !wait_until<20>([&] { return (int32_t)(*((volatile uint32_t*)&sm.prep_done[seq % PIPE_PREP_TEAMS]) - (seq - PIPE_RQ)) > 0; })) {
      *((volatile uint32_t*)&sm.v_err) = 1;
      return;
    }
    uint32_t ok = 1;
    if (lane == 0) {
      *((volatile uint32_t*)&sm.posting) = seq + 1;
      __threadfence_block();
      // in_use2 before in_use: the main warp takes over the builder's claim by setting in_use, then clearing in_use2
      const uint32_t victim = seq + 1 - PIPE_RQ;
      bool held = false;
      if (seq >= PIPE_RQ) {
        held = *((volatile uint32_t*)&sm.in_use2) == victim;
        __threadfence_block();
        held = held || *((volatile uint32_t*)&sm.in_use) == victim;
      }
      if (held) { *((volatile uint32_t*)&sm.posting) = 0; ok = 0; }
      else {
        sts_v4(&sm.rq_ent[seq % PIPE_RQ], cls, seq + 1, head, 0u);
        sts_u64(&sm.rq_word[seq % PIPE_RQ], ((unsigned long long)(seq + 1) << 32) | cls);
        // the slot's previous request (seq - PIPE_RING) was consumed by its prep team long ago (PIPE_RQ <= PIPE_RING)
        const unsigned long long tag = (unsigned long long)(seq + 1) << 32;
        st_relaxed_u64(&pg->req[seq % PIPE_RING][1], tag | head);
        st_relaxed_u64(&pg->req[seq % PIPE_RING][0], tag | cls);
        *((volatile uint32_t*)&sm.posting) = 0;
      }
    }
    if (__shfl_sync(FULL, ok, 0)) next_seq = seq + 1;
  };
  for (;;) {
    uint4 cw;
    while ((cw = lds_v4(&sm.cmd[tail % PIPE_CMDS])).x != tail + 1) __nanosleep(40);
    const uint32_t kind = cw.y & 3u, a = cw.z, b = cw.w;
    if (kind == PCMD_WB) {
      // log entries [a, b): record -> global table, Used += cnt x Resreq (node_info.go:203), node id -> modlog
      for (uint32_t base = a; base < b; base += 32) {
        const uint32_t i = base + lane;
        if (i < b) {
          const uint32_t hi = i % PIPE_HOT, node = sm.hot_node[hi], cnt = sm.hot_cnt[hi];
          uint64_t* gt = S.tiles + (size_t)(node / TILE_NODES) * ((size_t)NC * TILE_NODES) + (node % TILE_NODES);
#pragma unroll
          for (uint32_t c = 0; c < NC; ++c) gt[(size_t)c * TILE_NODES] = sm.hot_rec[c][hi];
          const ClassRec& cr = S.classes[sm.hot_cls[hi]];
#pragma unroll
          for (uint32_t k = 0; k < R; ++k) {
            double u = S.node_used[(size_t)k * S.N + node];
            const double rq = cr.resreq[k];
            for (uint32_t z = 0; z < cnt; ++z) u = KB_DADD(u, rq);
            S.node_used[(size_t)k * S.N + node] = u;
          }
          st_release_u32(&S.modlog[i], node);       // this lane's stores above are performed before the entry
        }
      }
      __syncwarp();
      if (lane == 0) { st_release_u32(&pg->log_head, b); *((volatile uint32_t*)&sm.pub_head) = b; }
    } else if (kind == PCMD_PLAN) {
      // planner: scan requests for the class of the next visit (a; PLAN_FORCE = whatever the table holds) and for the classes
      // of the runs after it in the static order of the next job's queue.  b = the log position the next visit starts from
      // (published: the visit's write-back command precedes this one).
      const uint32_t force = cw.y & PLAN_FORCE_BIT, head = b;
      uint32_t pc[KB_CHAIN_MAX];
      pc[0] = a;
      {
        const uint32_t s1 = S.job_pos[cw.y >> 3];
#pragma unroll
        for (uint32_t k = 0; k + 1 < KB_CHAIN_MAX; ++k) pc[k + 1] = S.ord_chain[(size_t)s1 * (KB_CHAIN_MAX - 1) + k];
      }
#pragma unroll
      for (uint32_t k = 0; k < KB_CHAIN_MAX; ++k) {
        const uint32_t pcls = pc[k];
        if (pcls == 0xFFFFFFFFu) continue;
        if (k == 0 && force) { post(pcls, head); continue; }
        const uint32_t amax = k == 0 ? PIPE_PATCH : ((S.pipe_pad >> (8u * k)) & 255u);
        if (amax == 255u) continue;
        uint32_t s2 = 0, st2 = 0;
        const bool f = rq_find<NC>(sm, lane, pcls, s2, st2);
        const bool pref = pref_class<PREF>(S, pcls);
        if (pref && k != 0) continue;      // only a list of the table state at its use will do: nothing further ahead
        if (!(f && list_usable(head, st2, amax, 0u, pref))) post(pcls, head);
      }
    } else {   // PCMD_QUIT
      if (lane == 0) { st_release_u32(&pg->quit, 1u); sm.n_requests = next_seq; __threadfence_block(); *((volatile uint32_t*)&sm.cmd_tail) = tail + 1; }
      return;
    }
    tail += 1;
    __syncwarp();
    if (lane == 0) { *((volatile uint32_t*)&sm.cmd_tail) = tail; dbg_put(S.dbg, 12, tail); }
  }
}

template <int RR, int WW, int PREF>
__device__ __forceinline__ void pipe_replayer(const DevSession& S, unsigned char* smem_raw) {
  constexpr uint32_t R = RR, W = WW, NC = 2 * RR + 6 + 3 * WW;
  using RS = ReplaySmem<NC>;
  RS& sm = *reinterpret_cast<RS*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  PipeG* pg = S.pg;
  Ctl* gctl = S.ctl;
  if (warp == 0) {
    load_ctl(sm.ctl, gctl, lane);
    if (lane < (int)PIPE_RQ) { sm.rq_ent[lane] = make_uint4(0u, 0u, 0u, 0u); sm.pb_ready[lane] = 0; sm.rq_word[lane] = 0ull; }
    for (uint32_t i = lane; i < PIPE_CMDS; i += 32) sm.cmd[i] = make_uint4(0u, 0u, 0u, 0u);
    if (lane < PIPE_PREP_TEAMS) sm.prep_done[lane] = (uint32_t)lane;
    if (lane == 0) {
      sm.cmd_tail = 0; sm.in_use = 0; sm.posting = 0; sm.n_requests = 0; sm.pub_head = 0; sm.v_quit = 0; sm.v_err = 0; sm.v_count = 0; sm.ext_slot = 0xFFFFFFFFu;
      sm.in_use2 = 0; sm.v_buf = 0; sm.b_gen = 0; sm.b_done = 0; sm.b_ring = 0;
    }
  }
  __syncthreads();
  int role, ridx;
  pipe_role(warp, role, ridx);
  if (role == ROLE_PATCH) { pipe_patch_warp<RR, WW, PREF>(S, sm, ridx, lane); return; }
  if (role == ROLE_PREP) { pipe_prep_warp<RR, WW, PREF>(S, sm, ridx / PIPE_PREP_TW, ridx % PIPE_PREP_TW, lane); return; }
  if (role == ROLE_WRITER) { pipe_writer_warp<RR, WW, PREF>(S, sm, lane); return; }
  if (role == ROLE_SHADOW) { pipe_shadow_warp<NC>(S, sm, lane); return; }
  if (role != ROLE_MAIN) return;

  // ---------------- main warp ----------------
  Ctl& c = sm.ctl;
  uint32_t priv_head = 0;        // log entries appended (the writer publishes them a little later)
  uint32_t cmd_head = 0;
  uint32_t fresh_floor = 0;      // after a rescan stop: only a list requested at or after this log position will do
  bool failed = false;
  // the latest build of the next chain's pool (its descriptor stays in sm.b_*): 0 none, B_LIVE published by the latest run and
  // not yet taken or dropped, B_DROPPED dropped and the builder perhaps not yet out of it
  constexpr uint32_t B_LIVE = 1, B_DROPPED = 2;
  uint32_t b_state = 0;
  auto push_cmd = [&](uint32_t kind, uint32_t a, uint32_t b) {       // whole warp calls it
    while (cmd_head - *((volatile uint32_t*)&sm.cmd_tail) >= PIPE_CMDS) __nanosleep(20);
    if (lane == 0) sts_v4(&sm.cmd[cmd_head % PIPE_CMDS], cmd_head + 1, kind, a, b);
    cmd_head += 1;
  };
  const bool timing = (S.pipe_pad & 1u) != 0;       // KB_PIPE_TIMING=1: clock64 phase timers of the main warp (kb_stats.cyc_*)
  auto err = [&] { return *((volatile uint32_t*)&sm.v_err) != 0; };      // another warp failed the cycle: a wait gives up
  // drop the live build without waiting for it: the builder stops at its next look at b_abort (visit start: the pool does not fit
  // this visit; otherwise the chain went on or the cycle ended)
  auto drop_build = [&](const bool at_visit_start) {
    if (lane == 0) {
      *((volatile uint32_t*)&sm.b_abort) = 1;
      if (timing) { if (at_visit_start) c.pipe_builds_missed += 1; else c.pipe_builds_cancelled += 1; }
    }
    b_state = B_DROPPED;
  };
  // before the patch warps, the hot ring or the descriptor are used again: wait until the builder has left a dropped build, then
  // release the list it may have claimed
  auto settle_build = [&]() {
    if (b_state != B_DROPPED) return;
    if (!wait_until<20>([&] { return *((volatile uint32_t*)&sm.b_done) == sm.b_gen; })) failed = true;
    if (lane == 0) *((volatile uint32_t*)&sm.in_use2) = 0;
    b_state = 0;
  };
  // the first visit's list
  if (!c.done) push_cmd(PCMD_PLAN | PLAN_FORCE_BIT | ((uint32_t)c.cur_job << 3), c.cur_class, 0u);
  uint32_t plan_idx = cmd_head;       // commands pushed up to and including the latest PCMD_PLAN

  if (lane == 0) sm.t_cycle0 = clock64();
  while (!c.done && !failed) {
    const uint32_t cls_id = c.cur_class;
    const long long t_v0 = timing ? clock64() : 0;
    if (lane == 0) { *((volatile uint32_t*)&sm.v_count) = sm.v_count + 1; dbg_put(S.dbg, 0, sm.v_count); dbg_put(S.dbg, 1, 1u); dbg_put(S.dbg, 2, cls_id); }       // wakes the shadow warp
    // ---------------- visit start: which list ----------------
    uint32_t seq = 0, stamp = 0;
    uint64_t cur_key = 0, floor_key = 0;
    uint32_t slot = 0;
    bool built = false;
    if (b_state == B_LIVE) {
      // the pool the builder prepared while the previous chain ended: usable iff this visit has the predicted class and starts
      // at the log head it was built for
      if (cls_id == sm.b_cls && sm.b_head == priv_head) {
        // sleeps between polls: the builder's warps share this warp's scheduler
        if (!wait_until<20>([&] { return *((volatile uint32_t*)&sm.b_done) == sm.b_gen; }, err)) { failed = true; break; }
        compiler_fence();
        built = sm.b_ok != 0;
      }
      if (built) {
        b_state = 0;
        seq = sm.b_seq; stamp = sm.b_lstamp;
        cur_key = sm.b_key[lane]; slot = sm.b_slot[lane]; floor_key = sm.b_floor;
        if (lane == 0) {
          sm.v_buf = sm.b_buf;
          *((volatile uint32_t*)&sm.in_use) = seq + 1;        // take over the builder's claim (the planner reads in_use2 first)
          __threadfence_block();
          *((volatile uint32_t*)&sm.in_use2) = 0;
          const uint32_t np = sm.b_npatch;
          if (np) { c.pipe_patched += 1; c.pipe_patch_entries += np; c.pairs_replayed += (unsigned long long)__popc(sm.b_pvalid); }
          c.pipe_urgent += sm.b_urgent;
          if (timing) { c.pipe_builds_used += 1; c.mispredictions += sm.b_waited; }
        }
        __syncwarp();
      } else drop_build(true);
    }
    if (!built) {
      const bool pref = pref_class<PREF>(S, cls_id);
      // The planner judged the table by the same rule when it handled this visit's PCMD_PLAN, or will in a moment: if nothing
      // usable is there yet, wait for it to get that far and look again.
      for (bool waited = false;;) {
        bool usable = rq_find<NC>(sm, lane, cls_id, seq, stamp);
        usable = usable && list_usable(priv_head, stamp, PIPE_PATCH, fresh_floor, pref);
        if (usable && claim(sm, &sm.in_use, seq, lane)) break;
        if (waited) {
          // its request stepped back: ask again, after a dropped build has let go of the list the planner has to recycle for it
          settle_build();
          if (failed) break;
          push_cmd(PCMD_PLAN | PLAN_FORCE_BIT | ((uint32_t)c.cur_job << 3), cls_id, priv_head), plan_idx = cmd_head;
        } else if (lane == 0) c.pipe_urgent += 1;
        if (!wait_until<20>([&] { return (int32_t)(*((volatile uint32_t*)&sm.cmd_tail) - plan_idx) >= 0; }, err)) { failed = true; break; }
        waited = true;
      }
      if (failed) break;
      const uint32_t pbi = seq % PIPE_RQ;
      if (lane == 0) { dbg_put(S.dbg, 1, 2u); dbg_put(S.dbg, 3, seq); dbg_put(S.dbg, 4, stamp); dbg_put(S.dbg, 5, priv_head); dbg_put(S.dbg, 6, cmd_head); }
      {
        const long long t_b0 = timing ? clock64() : 0;
        auto ready = [&] { return *((volatile uint32_t*)&sm.pb_ready[pbi]) == seq + 1; };
        if (timing && lane == 0 && !ready()) c.mispredictions += 1;      // visits that waited for their list (timing mode only)
        if (!wait_until<0>(ready, err)) failed = true;      // on the critical path: no sleep
        compiler_fence();          // pb[pbi] was stored before pb_ready by its team (fence + barrier on their side)
        if (timing && lane == 0) c.cyc_total += (unsigned long long)(clock64() - t_b0);      // timing mode: the wait for the prepared list
      }
      if (failed) break;
      const PrepBuf<NC>& P = sm.pb[pbi];
      settle_build();
      if (failed) break;
      if (lane == 0) sm.v_buf ^= 1u;
      __syncwarp();
      // patch set: log entries [stamp, priv_head)
      const uint32_t npatch = priv_head - stamp;
      uint32_t pn = 0;
      if (npatch) {
        const unsigned pvalid = __ballot_sync(FULL, patch_set(sm, stamp, npatch, pn, lane));
        sm.pnode[lane] = pn;
        if (lane == 0) {
          sm.v_pb = pbi; sm.v_stamp = stamp; sm.v_npatch = npatch; sm.v_pvalid = pvalid; sm.v_mode = 0;
          c.pipe_patched += 1; c.pipe_patch_entries += npatch; c.pairs_replayed += (unsigned long long)__popc(pvalid);
        }
        __syncwarp();
        if (lane == 0) dbg_put(S.dbg, 1, 3u);
        bar_sync(1, (1 + PIPE_PDEPTH) * 32);        // go: the patch warps evaluate depths 0..3 of the modified nodes
      }
      // ---------------- meanwhile: the prepared list minus the modified nodes, compacted (order is kept) ----------------
      floor_key = pool_complete(sm, P, pn, npatch, sm.cmp_key, sm.cmp_slot, cur_key, slot, lane,
                                [] { bar_sync(1, (1 + PIPE_PDEPTH) * 32); });      // done: the patch warps' keys are in place
    }
    fresh_floor = 0;
    const uint32_t pbi = seq % PIPE_RQ;
    const PrepBuf<NC>& P = sm.pb[pbi];
    const long long t_v1 = timing ? clock64() : 0;
    if (lane == 0) dbg_put(S.dbg, 1, 4u);
    // ---------------- pool -> 32 lane-owned candidates ----------------
    const bool have = cur_key != 0;
    const uint32_t my_node = key_node(cur_key);
    const uint32_t my_h = slot >> 5, my_l = slot & 31u;
    uint32_t depth = 0;                        // placements made on MY candidate
    bool cur_fi = have && (((my_h ? sm.pfi[sm.v_buf][0] : P.fi[0]) >> my_l) & 1u);
    if (lane == 0) c.scans += 1;
    const uint32_t my_lim = my_h ? (uint32_t)PIPE_PDEPTH : (uint32_t)PIPE_DEPTH;      // depths evaluated up front for MY candidate
    // extension: the whole warp evaluates depths base .. base+31 of the owner's candidate
    auto extend = [&](const uint32_t owner) {
      const uint32_t oslot = __shfl_sync(FULL, slot, owner), odepth = __shfl_sync(FULL, depth, owner), onode = __shfl_sync(FULL, my_node, owner);
      uint64_t r2[NC];
      pool_rec(sm, P, stamp, oslot, r2);
      const uint32_t base = odepth + 1, target = base + (uint32_t)lane;
      for (uint32_t k = 0; k < target; ++k) advance_rec<RR, WW>(r2, P.cls);
      RegAcc acc{r2, R, W};
      bool f = false;
      uint64_t k2 = eval_pair<RR, WW>(S.cf, P.cls, acc, onode, &f);
      if (PREF && P.is_pref) k2 = add_pref_term(k2, (int64_t)S.w_nodeaff, (int64_t)pref_count(P.pref, acc, W), (int64_t)P.pmax);
      __syncwarp();
      sm.ext_key[lane] = k2;
      const unsigned fm = __ballot_sync(FULL, f);
      if (lane == 0) { sm.ext_fi = fm; sm.ext_slot = oslot; sm.ext_base = base; c.pipe_extends += 1; c.pairs_replayed += 32ull; }
      __syncwarp();
    };
    if (lane == 0) sm.ext_slot = 0xFFFFFFFFu;
    __syncwarp();
    // a12 countdown: feasible nodes that reach the max count; when the last one fills up every key of this list is stale
    const bool is_pref = PREF && P.is_pref != 0 && P.pmax > 0;
    const int32_t my_cnt = (is_pref && have && my_h == 0) ? P.cnt[my_l] : -1;
    uint32_t nmax_live = P.pnmax;
    bool pref_stale = false;

    // Look-ahead of MY candidate: key / fits-idle of its NEXT state, kept in registers so that the owner of a pick moves on
    // without touching memory; the refill (a shared-memory read) is off the loop's dependency chain.
    const uint64_t* my_chain = my_h ? &sm.pkey[sm.v_buf][0][my_l] : &P.key[0][my_l];      // + d * KTOP: depth d
    const uint32_t* my_fiw = my_h ? &sm.pfi[sm.v_buf][0] : &P.fi[0];
    uint64_t next_key = 0;
    bool next_fi = false, have_next = false;
    auto refill = [&]() {                      // state at depth + 1, from the chain evaluated up front or the extension buffer
      const uint32_t dd = depth + 1;
      if (dd < my_lim) { next_key = my_chain[(size_t)dd * KTOP]; next_fi = ((my_fiw[dd] >> my_l) & 1u) != 0; have_next = true; }
      else if (sm.ext_slot == slot && dd >= sm.ext_base && dd < sm.ext_base + 32u) {
        next_key = sm.ext_key[dd - sm.ext_base]; next_fi = ((sm.ext_fi >> (dd - sm.ext_base)) & 1u) != 0; have_next = true;
      } else have_next = false;
    };
    refill();

    bool rescanned = false;
    for (;;) {              // runs of this class (consecutive visits of one class share the pool)
      if (c.done || c.cur_class != cls_id || (PREF && pref_stale)) break;
      const uint32_t j = (uint32_t)c.cur_job;
      const uint32_t q = c.cur_queue;
      const uint32_t jend = S.job_ord_off[j + 1];
      uint32_t run_left = c.cur_run;
      uint32_t placed = 0, popped = 0, n_alloc = 0;
      uint32_t reason = STOP_RUN_DONE;
      const uint32_t pos0 = __shfl_sync(FULL, lane == 0 ? S.job_pos[j] : 0u, 0);
      int32_t ready = 0, min_avail = 0;
      if (lane == 0) { ready = S.job_ready[j]; min_avail = S.job_min_avail[j]; }
      ready = __shfl_sync(FULL, ready, 0); min_avail = __shfl_sync(FULL, min_avail, 0);
      double jalloc = 0.0, qalloc = 0.0, my_rq = 0.0;
      if ((uint32_t)lane < R) {
        my_rq = P.cls.resreq[lane];
        if (S.drf_present) jalloc = S.job_alloc[(size_t)lane * S.J + j];
        if (S.proportion_present) qalloc = S.q_allocated[(size_t)lane * S.Q + q];
      }
      const uint32_t step0 = c.step;
      // The step loop carries ONE dependency chain (current keys -> arg-max -> owner -> the owner's next chain key); everything a
      // placement leaves behind — the decision record, the drf / proportion sums — is written after the loop, one lane per step.
      uint32_t flushed = 0;
      auto flush = [&](const uint32_t upto) {          // decisions of steps [flushed, upto), upto - flushed <= 32
        const uint32_t sidx = flushed + (uint32_t)lane;
        const bool act = sidx < upto;
        const uint32_t rec = act ? sm.step_rec[sidx & 31u] : 0u;
        const uint32_t nd = __shfl_sync(FULL, my_node, (int)(rec & 31u));
        if (act) {
          kb_decision dd;
          dd.node = (int32_t)nd;
          dd.kind = (rec & 32u) ? KB_KIND_ALLOCATED : KB_KIND_PIPELINED;
          dd.dispatched = 0; dd.reserved = 0;
          dd.step = step0 + sidx;
          dd.dispatch_step = 0xFFFFFFFFu;
          S.dec[S.ord_task[pos0 + sidx]] = dd;
        }
        flushed = upto;
        __syncwarp();
      };
      const long long t_run0 = timing ? clock64() : 0;
      while (run_left > 0) {      // steps: one pending task each (allocate.go:129-189)
        const uint64_t best = warp_max_u64(cur_key);
        if (best < floor_key) { reason = STOP_RESCAN; break; }
        popped += 1;
        run_left -= 1;
        if (best == 0) { reason = STOP_NOFIT; break; }              // allocate.go:144-148
        const uint32_t owner = (uint32_t)__ffs(__ballot_sync(FULL, cur_key == best)) - 1u;
        const bool fits_idle = ((__ballot_sync(FULL, cur_fi) >> owner) & 1u) != 0;
        const bool own = (uint32_t)lane == owner;
        if (__any_sync(FULL, own && !have_next)) { extend(owner); if (own) refill(); }      // rare: chain exhausted
        bool left_max = false;
        if (own) {                                 // ssn.Allocate / ssn.Pipeline: my candidate moves to its next state
          depth += 1;
          cur_key = next_key;
          cur_fi = next_fi;
          if (PREF) left_max = is_pref && cur_key == 0 && my_cnt == (int32_t)P.pmax;      // a max-count node left the feasible set
          refill();
        }
        if (lane == 0) sm.step_rec[placed & 31u] = owner | (fits_idle ? 32u : 0u);
        placed += 1;
        n_alloc += fits_idle ? 1u : 0u;
        if ((placed & 31u) == 0) { __syncwarp(); flush(placed); }
        if (PREF && is_pref && __any_sync(FULL, left_max)) { nmax_live -= 1; pref_stale = nmax_live == 0; }
        const bool jr = !S.gang_ready || (ready + (int32_t)n_alloc) >= min_avail;     // ssn.JobReady
        if (jr && (pos0 + popped < jend)) { reason = STOP_YIELD; break; }             // allocate.go:185-188
        if (PREF && pref_stale) { if (run_left > 0) reason = STOP_RESCAN; break; }
      }
      const long long t_loop1 = timing ? clock64() : 0;
      __syncwarp();
      // this run may end the chain: the builder starts on the next chain's pool now, the bookkeeping below runs meanwhile.  The
      // class of the next chain is the planner's prediction (ord_chain, the queue's static job order); with several queues the
      // queue heap reorders the visits, the prediction mostly misses and a build would only take issue slots from this warp
      const uint32_t nxt = S.Q == 1 ? __shfl_sync(FULL, lane == 0 ? S.ord_chain[(size_t)pos0 * (KB_CHAIN_MAX - 1)] : 0u, 0) : 0xFFFFFFFFu;
      if (reason != STOP_RESCAN && !(PREF && pref_stale) && nxt != 0xFFFFFFFFu) {
        settle_build();
        const unsigned mm = __ballot_sync(FULL, depth > 0);
        sm.b_mnode[lane] = my_node; sm.b_mslot[lane] = depth > 0 ? (slot | (depth << 8)) : 0u;
        if (lane == 0) {
          sm.b_gen += 1; sm.b_cls = nxt; sm.b_ccls = cls_id; sm.b_head = priv_head + (uint32_t)__popc(mm); sm.b_pb = pbi; sm.b_stamp = stamp;
          sm.b_buf = sm.v_buf ^ 1u;
          *((volatile uint32_t*)&sm.b_plan) = 0; *((volatile uint32_t*)&sm.b_abort) = 0; sm.v_mode = 1;
        }
        __syncwarp();
        bar_arrive(1, (1 + PIPE_PDEPTH) * 32);      // go, without waiting for the builder
        b_state = B_LIVE;
      }
      if (flushed < placed) flush(placed);
      for (uint32_t z = 0; z < placed; ++z) { jalloc = KB_DADD(jalloc, my_rq); qalloc = KB_DADD(qalloc, my_rq); }      // AllocateFunc handlers, in order
      if (lane == 0) {
        S.job_pos[j] = pos0 + popped;
        S.job_ready[j] = ready + (int32_t)n_alloc;
        S.job_placed[j] += placed;
        c.step = step0 + placed;
        c.tasks_processed += popped;
        c.pairs_logical += (unsigned long long)popped * S.N;
        c.tasks_allocated += n_alloc;
        c.tasks_pipelined += placed - n_alloc;
      }
      if ((uint32_t)lane < R && placed) {
        if (S.drf_present) S.job_alloc[(size_t)lane * S.J + j] = jalloc;
        if (S.proportion_present) S.q_allocated[(size_t)lane * S.Q + q] = qalloc;
      }
      if (placed) {        // drf.calculateShare (lanes 0..R-1) and proportion.updateShare (lanes 8..8+R-1): all divisions side by side
        const int k8 = lane & 7;
        const double qa = __shfl_sync(FULL, qalloc, k8);
        double v = 0.0;
        if (lane < 8) {
          if (S.drf_present && (uint32_t)lane < R && ((S.total_dims_mask >> lane) & 1u)) v = share_of(jalloc, S.total[lane]);
        } else if (lane < 16) {
          if (S.proportion_present && (uint32_t)k8 < R) {
            const uint32_t present = S.q_deserved_present[q] | 3u;
            if ((present >> k8) & 1u) v = share_of(qa, S.q_deserved[(size_t)k8 * S.Q + q]);
          }
        }
        const uint64_t m1 = warp_max_u64(lane < 8 ? double_as_u64(v) : 0ull);
        const uint64_t m2 = warp_max_u64((lane >= 8 && lane < 16) ? double_as_u64(v) : 0ull);
        if (lane == 0) {
          if (S.drf_present) S.job_share[j] = u64_as_double(m1);
          if (S.proportion_present) S.q_share[q] = u64_as_double(m2);
        }
      }
      __syncwarp();
      const long long t_run1 = timing ? clock64() : 0;
      if (lane == 0) {
        if (reason == STOP_RESCAN) c.rescans += 1;
        after_run<0>(S, c, reason, placed, true);
        if (timing) {
          const long long t_run2 = clock64();
          c.cyc_steps += (unsigned long long)(t_run1 - t_run0);
          c.cyc_merge += (unsigned long long)(t_loop1 - t_run0);      // the step loop alone
          c.cyc_ctl += (unsigned long long)(t_run2 - t_run1);
          c.predictions += 1;               // runs (timing mode only)
        }
      }
      __syncwarp();
      if (reason == STOP_RESCAN) { rescanned = true; break; }
      if (b_state == B_LIVE && !(c.done || c.cur_class != cls_id || (PREF && pref_stale))) drop_build(false);      // the chain goes on

    }

    if (lane == 0) { dbg_put(S.dbg, 1, 5u); dbg_put(S.dbg, 7, c.rescans); }
    const long long t_r0 = timing ? clock64() : 0;
    // ---------------- end of the visit chain on this class: modified candidates -> hot ring + log ----------------
    const uint32_t nmod = (uint32_t)__popc(__ballot_sync(FULL, depth > 0));
    if (nmod && b_state == B_LIVE) {
      // the builder has put these records into the ring (pipe_build)
      if (!wait_until<0>([&] { return *((volatile uint32_t*)&sm.b_ring) == sm.b_gen; }, err)) failed = true;
      compiler_fence();
    } else if (nmod) {
      settle_build();
      if (!ring_append<RR, WW>(sm, P, stamp, priv_head + nmod, slot, depth, my_node, cls_id, lane)) failed = true;
    }
    if (failed) break;
    if (nmod) {
      __syncwarp();
      push_cmd(PCMD_WB, priv_head, priv_head + nmod);
      priv_head += nmod;
    }
    if (rescanned) fresh_floor = priv_head;
    if (lane == 0) *((volatile uint32_t*)&sm.in_use) = 0;          // P is not read past this point
    // the planner (writer warp) requests the lists of the next visits, stamped with the log position this visit ended at
    // (pushing this before the write-back command, with the stamp ahead of the published log, was measured slower on C3)
    if (!c.done) {
      push_cmd(PCMD_PLAN | (rescanned ? PLAN_FORCE_BIT : 0u) | ((uint32_t)c.cur_job << 3), c.cur_class, priv_head); plan_idx = cmd_head;
      if (b_state == B_LIVE && lane == 0) *((volatile uint32_t*)&sm.b_plan) = plan_idx;
    }
    const long long t_r1 = timing ? clock64() : 0;
    if (lane == 0) dbg_put(S.dbg, 1, 6u);
    if (lane == 0 && timing) {
      const long long t_end = clock64();
      c.cyc_scan += (unsigned long long)(t_v1 - t_v0);
      c.cyc_replay += (unsigned long long)(t_end - t_v1);
      c.cyc_ring += (unsigned long long)(t_r1 - t_r0);
      c.cyc_plan += (unsigned long long)(t_end - t_r1);
    }
    __syncwarp();
  }

  // ---------------- wind down ----------------
  if (lane == 0) dbg_put(S.dbg, 1, 7u);
  if (b_state == B_LIVE) drop_build(false);
  settle_build();
  if (lane == 0) { *((volatile uint32_t*)&sm.v_quit) = 1; }
  __syncwarp();
  bar_sync(1, (1 + PIPE_PDEPTH) * 32);           // releases the patch warps
  push_cmd(PCMD_QUIT, 0, 0);
  if (!wait_until<40>([&] { return *((volatile uint32_t*)&sm.cmd_tail) == cmd_head; })) failed = true;
  if (lane == 0) {
    if (!timing) c.cyc_total += (unsigned long long)(clock64() - sm.t_cycle0);
    const uint32_t n_requests = *((volatile uint32_t*)&sm.n_requests);
    c.pipe_requests += n_requests; c.pairs_scanned += (unsigned long long)n_requests * S.N;
    if ((failed || *((volatile uint32_t*)&sm.v_err)) && !c.error) c.error = 3;
    const uint32_t perr = ld_relaxed_u32(&pg->error);
    if (perr && !c.error) c.error = perr;
  }
  __syncwarp();
  store_ctl(gctl, c, lane);
}

// PREF: the session has classes with preferred node-affinity terms (a12); 0 compiles the two-pass scan, the fresh-list rule and
// the max-count countdown out of the hot paths
template <int RR, int WW, int PREF>
__global__ void __launch_bounds__(PIPE_THREADS, 1)
cycle_kernel(const __grid_constant__ DevSession S) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  if (blockIdx.x == gridDim.x - 1) pipe_replayer<RR, WW, PREF>(S, smem_raw);
  else pipe_scanner<RR, WW, PREF>(S, smem_raw);
}

}  // namespace kb
