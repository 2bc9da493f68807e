// kb_core.h — host/device-shared core of the engine: the exact per-(task,node) arithmetic
// (K1 predicate bitmask + K2 fused score -> packed key) and the small resource algebra the
// commit path needs.  Everything here is `KB_HD` so the very same code is compiled by nvcc
// into the kernels and by g++ into tests/emu (logic tests without a GPU).
//
// Semantics follow the reference (paths relative to kube-batch/pkg/scheduler):
//   resource fit      actions/allocate/allocate.go:73-87 + api/resource_info.go:268-302 (LessEqual)
//   predicates        plugins/predicates/predicates.go:123-265 + vendored predicates.go
//   node scores       vendor/k8s.io/kubernetes/pkg/scheduler/algorithm/priorities/{least_requested,
//                     most_requested,balanced_resource_allocation,resource_allocation}.go
//   score sum         util/scheduler_helper.go:162-168
//   best node         util/scheduler_helper.go:188-208 with the deterministic first-max rule
//
// FP64 fidelity: Go on amd64 never fuses a*b+c, so every product / quotient that feeds a
// decision goes through KB_DMUL / KB_DDIV / KB_DSUB (round-to-nearest intrinsics on device,
// plain operators compiled with -ffp-contract=off on host).
#ifndef KB_CORE_H_
#define KB_CORE_H_

#include <stdint.h>
#include "../../include/kbgpu.h"

#if defined(__CUDACC__)
#define KB_HD __host__ __device__ __forceinline__
#else
#define KB_HD inline
#endif

#if defined(__CUDA_ARCH__)
#define KB_DSUB(a, b) __dsub_rn((a), (b))
#define KB_DMUL(a, b) __dmul_rn((a), (b))
#define KB_DDIV(a, b) __ddiv_rn((a), (b))
#define KB_DADD(a, b) __dadd_rn((a), (b))
#define KB_FABS(a) fabs(a)
#define KB_LL2D(a) __ll2double_rn(a)
#define KB_D2LL(a) __double2ll_rz(a)
#else
#include <math.h>
#define KB_DSUB(a, b) ((a) - (b))
#define KB_DMUL(a, b) ((a) * (b))
#define KB_DDIV(a, b) ((a) / (b))
#define KB_DADD(a, b) ((a) + (b))
#define KB_FABS(a) fabs(a)
#define KB_LL2D(a) ((double)(a))
#define KB_D2LL(a) ((long long)(a))
#endif

namespace kb {

// api/resource_info.go:68-70
#define KB_MIN_MILLI_CPU 10.0
#define KB_MIN_MILLI_SCALAR 10.0
#define KB_MIN_MEMORY (10.0 * 1024.0 * 1024.0)

constexpr int KTOP = 32;          // candidates kept per class per scan (one warp-wide sorted list)
constexpr int DMAX = 32;          // dirty nodes a replay epilogue can hold
constexpr int TILE_NODES = 128;   // nodes per TMA tile (== threads per scan CTA)

// Job-order comparators in tier/plugin order (framework/session_plugins.go:243-267)
enum JobCmp : uint32_t { JOBCMP_NONE = 0, JOBCMP_PRIORITY = 1, JOBCMP_GANG = 2, JOBCMP_DRF = 3 };

// Resolved plugin configuration: what OnSessionOpen of the built-in plugins registers, by name.
struct EvalConf {
  uint32_t R, W;
  uint32_t predicates;        // predicates plugin registered && EnabledPredicate
  uint32_t mem_pressure, disk_pressure, pid_pressure;   // predicates.go:33-40 arguments
  uint32_t nodeorder;         // nodeorder plugin registered && EnabledNodeOrder
  int32_t  w_least, w_most, w_balanced;                 // nodeorder.go:107-131 (node/pod-affinity terms are 0 here)
  int64_t  score_bias;        // makes the weighted sum non-negative so it packs into the key
  uint32_t fit_mode;          // 0: allocate — InitResreq <= Idle || InitResreq <= Releasing (allocate.go:82)
                              // 1: backfill — no resource predicate, but NodeInfo.AddTask needs Resreq <= Idle
                              //    (node_info.go:161-167): the backfill view's class table carries Resreq in `initreq`
                              //    and the Releasing alternative is masked off
                              // 2: backfill with the predicates plugin enabled — the key ignores the resources altogether: the
                              //    task goes to the FIRST node that passes ssn.PredicateFn, and if node.AddTask refuses it there
                              //    the task stays Allocated on no node and every later predicate of the session fails
                              //    (Ctl.pred_dead); `fits_idle` still reports Resreq <= Idle
  uint32_t pad0;
};

// One task equivalence class: every field of a pending task that predicateFn / the prioritizers /
// AddTask read.  Tasks of a PodGroup are normally one class.
struct ClassRec {
  double   initreq[KB_MAX_R];
  double   resreq[KB_MAX_R];
  int64_t  nz_cpu, nz_mem;
  uint64_t sel_req[KB_MAX_W];
  uint64_t aff[KB_MAX_AFF_TERMS][KB_MAX_W];
  uint64_t tol[KB_MAX_W];
  uint64_t port_own[KB_MAX_W];
  uint64_t port_conflict[KB_MAX_W];
  uint64_t aff_own[KB_MAX_W];     // bits an ALLOCATE placement (not a Pipeline) adds to the node's port words: host-level inter-pod
                                  // anti-affinity encoded as atoms (kb_build.h affinity_as_atoms); all zero otherwise
  uint32_t n_aff;
  uint32_t flags;             // KB_TASK_BEST_EFFORT_QOS only
};

// Preferred node-affinity terms of a class (NodeAffinityPriority, vendor/.../priorities/node_affinity.go:34-77): requirement
// atoms that must ALL hold on the node + the term's weight.  Evaluated by cycle_kernel (two-pass scan, kb_pipe.cuh), the
// per-visit kernels (kb_kernels.cuh), preempt's sweep (kb_evict.h) and the emulation.
struct ClassPref {
  uint64_t term[KB_MAX_PREF_TERMS][KB_MAX_W];
  int32_t  weight[KB_MAX_PREF_TERMS];
  uint32_t n;
  uint32_t pad[3];
};

// api/resource_info.go:268-274: `l < r || math.Abs(l-r) < diff`.  Evaluated as ONE rounded subtraction and ONE compare:
//   l <  r  ->  l - r < 0 < diff (a difference of distinct doubles never rounds to zero: gradual underflow), true either way;
//   l >= r  ->  |l - r| == l - r, the same rounded value the reference compares.
// (NaN never occurs: quantities are finite; +-inf from an overflowing subtraction compares like the reference's.)
// Pinned against the two-term form over the reference's LessEqual vectors and random values in tests/test_emu_parity.py.
KB_HD bool le_func(double l, double r, double diff) { return KB_DSUB(l, r) < diff; }
KB_HD bool le_func_reference_form(double l, double r, double diff) { return l < r || KB_FABS(KB_DSUB(l, r)) < diff; }

// Resource.LessEqual(l, r) on dense vectors (api/resource_info.go:268-302).  A nil scalar map and a
// map of zeros are indistinguishable here: a scalar of l is only compared when l_k > 10, and then
// `rr == nil -> false` and `l_k < 0 || |l_k - 0| < 10` both yield false (DESIGN.md §dense resources).
template <class LAcc, class RAcc>
KB_HD bool res_less_equal(uint32_t R, LAcc l, RAcc r) {
  if (!le_func(l(0), r(0), KB_MIN_MILLI_CPU)) return false;
  if (!le_func(l(1), r(1), KB_MIN_MEMORY)) return false;
  for (uint32_t k = 2; k < R; ++k) {
    double lq = l(k);
    if (lq <= KB_MIN_MILLI_SCALAR) continue;
    if (!le_func(lq, r(k), KB_MIN_MILLI_SCALAR)) return false;
  }
  return true;
}

// api/resource_info.go:93-105
template <class Acc>
KB_HD bool res_is_empty(uint32_t R, Acc v) {
  if (!(v(0) < KB_MIN_MILLI_CPU && v(1) < KB_MIN_MEMORY)) return false;
  for (uint32_t k = 2; k < R; ++k)
    if (v(k) >= KB_MIN_MILLI_SCALAR) return false;
  return true;
}

// api/helpers/helpers.go:47-60
KB_HD double share_of(double l, double r) {
  if (r == 0) return l == 0 ? 0.0 : 1.0;
  return KB_DDIV(l, r);
}

// a / b (Go int64 division) for b > 0 when the quotient is known to lie in [0, 10] — no 64-bit integer division (hundreds
// of cycles on the GPU), no ten-step ladder: a single-precision estimate (relative error < 2^-21, so |est - a/b| < 1e-5)
// and ONE exact multiply-compare fix-up in each direction.  Exact for every 0 <= a <= 10 b, b < 2^59.
KB_HD int64_t div_0_to_10(int64_t a, int64_t b) {
  if (a < 0 || a > 10 * b) return a / b;          // outside the fast range (never on sane inputs)
#if defined(__CUDA_ARCH__)
  int64_t q = (int64_t)__float2int_rz(__fdividef(__ll2float_rn(a), __ll2float_rn(b)));     // MUFU.RCP + FMUL
#else
  int64_t q = (int64_t)((float)a * (1.0f / (float)b));
#endif
  q = q < 0 ? 0 : (q > 10 ? 10 : q);
  q -= (q * b > a) ? 1 : 0;
  q += ((q + 1) * b <= a) ? 1 : 0;
  return q;
}
// least_requested.go:49-58
KB_HD int64_t least_requested_score(int64_t requested, int64_t capacity) {
  if (capacity == 0) return 0;
  if (requested > capacity) return 0;
  if (capacity < 0 || capacity > ((int64_t)1 << 58)) return ((capacity - requested) * 10) / capacity;
  return div_0_to_10((capacity - requested) * 10, capacity);
}
// most_requested.go:52-61
KB_HD int64_t most_requested_score(int64_t requested, int64_t capacity) {
  if (capacity == 0) return 0;
  if (requested > capacity) return 0;
  if (capacity < 0 || capacity > ((int64_t)1 << 58)) return (requested * 10) / capacity;
  return div_0_to_10(requested * 10, capacity);
}
// balanced_resource_allocation.go:42-79 (BalanceAttachedNodeVolumes gate off)
KB_HD int64_t balanced_score(int64_t req_cpu, int64_t cap_cpu, int64_t req_mem, int64_t cap_mem) {
  double cf = cap_cpu == 0 ? 1.0 : KB_DDIV(KB_LL2D(req_cpu), KB_LL2D(cap_cpu));
  double mf = cap_mem == 0 ? 1.0 : KB_DDIV(KB_LL2D(req_mem), KB_LL2D(cap_mem));
  if (cf >= 1.0 || mf >= 1.0) return 0;
  double diff = KB_FABS(KB_DSUB(cf, mf));
  return (int64_t)KB_D2LL(KB_DMUL(KB_DSUB(1.0, diff), 10.0));
}

// NodeAffinityPriority Map (node_affinity.go:34-77): count = sum of the weights of the preferred terms whose requirement
// atoms ALL hold on the node (weight 0 terms are skipped)
template <class NodeAcc>
KB_HD int32_t pref_count(const ClassPref& cp, const NodeAcc& n, uint32_t W) {
  int32_t count = 0;
  for (uint32_t p = 0; p < cp.n && p < KB_MAX_PREF_TERMS; ++p) {
    if (cp.weight[p] == 0) continue;
    bool match = true;
    for (uint32_t w = 0; w < W; ++w) match = match && ((n.labels(w) & cp.term[p][w]) == cp.term[p][w]);
    if (match) count += cp.weight[p];
  }
  return count;
}
// ... and its Reduce, NormalizeReduce(MaxPriority = 10, reverse = false) (reduce.go:28-63) over the FEASIBLE nodes, times the
// nodeaffinity.weight: what the node's packed key gains.  max_count == 0: every score stays 0.
KB_HD uint64_t add_pref_term(uint64_t key, int64_t w_nodeaff, int64_t count, int64_t max_count) {
  if (!key || max_count <= 0) return key;
  const int64_t hi = (int64_t)(key >> 32) + w_nodeaff * (10 * count / max_count);
  return ((uint64_t)hi << 32) | (key & 0xFFFFFFFFull);
}

// Packed candidate key: (biased score << 32) | (0xFFFFFFFF - node).  max over keys == highest score,
// ties to the smallest canonical node index (== lexicographically smallest node name).  0 == infeasible.
KB_HD uint64_t pack_key(int64_t biased_score, uint32_t node) {
  return ((uint64_t)biased_score << 32) | (uint64_t)(0xFFFFFFFFu - node);
}
KB_HD uint32_t key_node(uint64_t key) { return 0xFFFFFFFFu - (uint32_t)(key & 0xFFFFFFFFull); }
KB_HD int64_t key_score(uint64_t key) { return (int64_t)(key >> 32); }

// K2 alone: the biased weighted sum of the Map priorities for one (class, node) pair (util/scheduler_helper.go:162-168)
template <class NodeAcc>
KB_HD int64_t node_score(const EvalConf& cf, const ClassRec& c, const NodeAcc& n) {
  int64_t score = cf.score_bias;
  if (cf.nodeorder) {
    // resource_allocation.go:100-123: req = nodeInfo.NonZeroRequest() + pod non-zero request
    const int64_t rc = n.nz_cpu() + c.nz_cpu, rm = n.nz_mem() + c.nz_mem;
    const int64_t ac = n.alloc_cpu(), am = n.alloc_mem();
    if (cf.w_least)    score += ((least_requested_score(rc, ac) + least_requested_score(rm, am)) / 2) * (int64_t)cf.w_least;
    if (cf.w_most)     score += ((most_requested_score(rc, ac) + most_requested_score(rm, am)) / 2) * (int64_t)cf.w_most;
    if (cf.w_balanced) score += balanced_score(rc, ac, rm, am) * (int64_t)cf.w_balanced;
  }
  return score;
}

// NodeAcc concept: idle(r) rel(r) -> double; alloc_cpu() alloc_mem() nz_cpu() nz_mem() -> int64_t;
// pods() max_pods() -> int32_t; flags() -> uint32_t; labels(w) taints(w) ports(w) -> uint64_t.
//
// K1 (predicate bitmask) + K2 (fused score) for one (class, node) pair against the node's CURRENT state.
// Returns the packed key, 0 if predicateFn would return an error.  `fits_idle` reports
// InitResreq <= Idle, which decides Allocate vs Pipeline at commit (allocate.go:160); `pred_ok` (optional) reports
// ssn.PredicateFn alone — backfill needs it to reproduce ssn.Allocate's status-before-AddTask order (session.go:241-262).
// RR / WW: compile-time copies of cf.R / cf.W (0 = read them at run time).  The kernels instantiate the common geometry
// (R = 3, W = 2) so that every loop below unrolls into straight-line code; semantics are identical.
template <int RR = 0, int WW = 0, class NodeAcc>
KB_HD uint64_t eval_pair(const EvalConf& cf, const ClassRec& c, const NodeAcc& n, uint32_t node_idx, bool* fits_idle, bool* pred_ok = nullptr) {
  // Written branch-free on purpose: a lone warp (the replay) or one warp per SM sub-partition (the scan)
  // hides latency only through instruction-level parallelism, so every check is computed and AND-ed.
  const uint32_t R = RR ? (uint32_t)RR : cf.R, W = WW ? (uint32_t)WW : cf.W;
  // allocate.go:82: !InitResreq.LessEqual(Idle) && !InitResreq.LessEqual(Releasing) -> ResourceFit failed
  bool fi = le_func(c.initreq[0], n.idle(0), KB_MIN_MILLI_CPU) & le_func(c.initreq[1], n.idle(1), KB_MIN_MEMORY);
  bool fr = le_func(c.initreq[0], n.rel(0), KB_MIN_MILLI_CPU) & le_func(c.initreq[1], n.rel(1), KB_MIN_MEMORY);
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
  for (uint32_t k = 2; k < R; ++k) {            // resource_info.go:286-299: scalars <= 10 are skipped
    const double lq = c.initreq[k];
    const bool skip = lq <= KB_MIN_MILLI_SCALAR;
    fi = fi & (skip | le_func(lq, n.idle(k), KB_MIN_MILLI_SCALAR));
    fr = fr & (skip | le_func(lq, n.rel(k), KB_MIN_MILLI_SCALAR));
  }
  fr = fr & (cf.fit_mode == 0);                 // backfill only ever allocates from Idle
  if (fits_idle) *fits_idle = fi;
  bool ok = fi | fr | (cf.fit_mode == 2);
  bool pok = true;            // ssn.PredicateFn alone (the predicates plugin), irrespective of the resource fit

  if (cf.predicates) {
    const uint32_t fl = n.flags();
    pok = pok & (n.max_pods() > n.pods());                                                             // predicates.go:127
    pok = pok & ((fl & (KB_NODE_NOT_READY | KB_NODE_NET_UNAVAILABLE | KB_NODE_UNSCHEDULABLE)) == 0);   // vendored :1675-1698
    uint64_t bad = 0;
    uint64_t miss[KB_MAX_AFF_TERMS] = {0, 0, 0, 0};
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (uint32_t w = 0; w < W; ++w) {
      const uint64_t lab = n.labels(w);
      bad |= (lab & c.sel_req[w]) ^ c.sel_req[w];          // nodeSelector atoms missing        (:927-935)
      bad |= n.ports(w) & c.port_conflict[w];              // host port conflict                 (:1153-1173)
      bad |= n.taints(w) & ~c.tol[w];                      // untolerated NoSchedule/NoExecute   (:1596-1624)
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
      for (uint32_t t = 0; t < KB_MAX_AFF_TERMS; ++t) miss[t] |= (lab & c.aff[t][w]) ^ c.aff[t][w];
    }
    pok = pok & (bad == 0);
    // required node affinity: OR of AND-terms (:944-968); unused term slots hold all-zero masks, so gate on n_aff
    bool any = c.n_aff == 0;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (uint32_t t = 0; t < KB_MAX_AFF_TERMS; ++t) any = any | ((t < c.n_aff) & (miss[t] == 0));
    pok = pok & any;
    const bool memp = cf.mem_pressure && (c.flags & KB_TASK_BEST_EFFORT_QOS) && (fl & KB_NODE_MEM_PRESSURE);   // :1633-1650
    const bool diskp = cf.disk_pressure && (fl & KB_NODE_DISK_PRESSURE);                                       // :1654-1660
    const bool pidp = cf.pid_pressure && (fl & KB_NODE_PID_PRESSURE);                                          // :1664-1671
    pok = pok & !(memp | diskp | pidp);
  }
  if (pred_ok) *pred_ok = pok;
  ok = ok & pok;

  return ok ? pack_key(node_score(cf, c, n), node_idx) : 0ull;
}

}  // namespace kb
#endif  // KB_CORE_H_
