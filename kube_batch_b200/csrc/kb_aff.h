// kb_aff.h — inter-pod (anti)affinity on the device: predicate step 10 (InterPodAffinityMatches) and InterPodAffinityPriority
// over the counters of include/kbgpu.h kb_pod_affinity.  Host/device shared (KB_HD): the kernels (kb_kernels.cuh), the host
// build (kb_build.h) and tests/emu compile the same functions.
//
// Reference (paths relative to kube-batch):
//   predicate   vendor/k8s.io/kubernetes/pkg/scheduler/algorithm/predicates/predicates.go:1261-1572 (slow path, meta == nil),
//               pods from pkg/scheduler/plugins/util/util.go:37-85 (AllocatedStatus tasks of the session's jobs)
//   priority    vendor/k8s.io/kubernetes/pkg/scheduler/algorithm/priorities/interpod_affinity.go:99-235 over the FEASIBLE nodes,
//               pods from NodeInfo.Tasks; pkg/scheduler/plugins/nodeorder/nodeorder.go:49-63 (node of a not-yet-bound pod)
//
// What moves during a cycle (all of it written by the ONE replaying thread, read by the scans of later launches):
//   cnt[g][domain], total[g]   members of counter group g — a task joins when ssn.Allocate places it (status Allocated is an
//                              AllocatedStatus; Pipelined is not, so ssn.Pipeline does not count)
//   kind_count[kind][node]     pods per kind in NodeInfo.Tasks — Allocate and Pipeline both call node.AddTask
//   first_unbound              lowest node index holding a pod with an empty Spec.NodeName — every pod placed in the session
// A placement can change the feasibility / score of EVERY node of a topology domain, so the "one node column changes per
// placement" rule behind the candidate lists (DESIGN.md §2) does not hold for a class whose keys read these counters: such a
// class (aff_stop_each) gets a fresh scan per task — the replay stops after one placement.  Exception: a class whose own
// placements only touch single-node domains (one replica per host) keeps its multi-task runs (ClassAff.pred_multi_ok).
#ifndef KB_AFF_H_
#define KB_AFF_H_

#include "kb_core.h"

// The counters are written by one launch and read by the next; visit_kernel may be scheduled (programmatic dependent launch)
// while its predecessor still runs, so an SM's L1 can hold a line the predecessor's scan read before its replay changed it:
// every read of MUTABLE affinity data goes to L2 (ld.global.cg), like the control block and the candidate lists.
#if defined(__CUDA_ARCH__)
#define KB_LDM(p) __ldcg(p)
#else
#define KB_LDM(p) (*(p))
#endif

namespace kb {

// A forbidden counter group >= 64 of a class, resolved by the host build so that the scan goes node_domain -> cnt directly.
struct AffX {
  uint32_t row;           // group_keyset[g] * N: the key set's row of node_domain
  uint32_t off;           // group_off[g]: the group's counters
};

// Groups 0..63 are bits of the masks; groups >= 64 (kb_pod_affinity.task_xgroup) sit in two packed per-class lists.
struct ClassAff {
  uint64_t forbid;        // groups < 64 whose members in the node's domain reject the node
  uint64_t contrib;       // groups < 64 the task joins once Allocated
  uint64_t w_keysets;     // key sets that appear in the class's weight list
  int32_t  need;          // group the required pod-affinity terms need, -1 none
  int32_t  kind;          // kind of the placed pod, -1 none
  uint32_t w_off, w_cnt;  // weight list (AffDev.w_*)
  uint16_t self_match;    // KB_TASK_AFF_SELF_MATCH
  uint16_t self_block;    // a placement of this class makes the chosen node infeasible for the class itself (one replica per host)
  uint32_t pred_multi_ok; // the predicate part of the class survives its OWN placements: the only counters it both joins and reads
                          // belong to key sets whose domains are single nodes (kubernetes.io/hostname), so a placement changes
                          // nothing but the chosen node — the candidate list stays exact and a run may place several tasks
  uint32_t xf_off, xf_cnt;  // forbidden groups >= 64: AffDev.xf[xf_off .. xf_off + xf_cnt); the first xs_cnt of them are also joined
  uint32_t xs_cnt;          //   (the groups aff_self_blocks reads)
  uint32_t xc_off, xc_cnt;  // joined groups >= 64: AffDev.xc[xc_off .. xc_off + xc_cnt) (group ids)
  uint32_t x_pad;
};

struct AffDev {
  uint32_t on;                    // the session carries kb_pod_affinity
  uint32_t n_keysets, n_groups, n_kinds;
  uint32_t has_weights;           // some class has a weight list: the priority passes run before every visit
  int32_t  w_podaff;              // podaffinity.weight (nodeorder.go:111-117)
  uint32_t dom_total;             // sum of the key sets' domain counts (size of dom_sum)
  uint32_t has_pref;              // some class carries preferred NODE-affinity terms and the session runs on the per-visit kernels:
                                  // pass 2 also reduces the max count over the feasible nodes (NodeAffinityPriority, minmax[2])
  uint32_t has_x;                 // some class names groups >= 64 (xf / xc lists): sessions without skip every list walk
  const int32_t*  node_domain;    // [n_keysets][N]
  const uint32_t* keyset_off;     // [n_keysets + 1] offsets into dom_sum
  const uint32_t* group_keyset;   // [n_groups]
  const uint32_t* group_off;      // [n_groups] offsets into cnt
  const ClassAff* cls;            // [C]
  const AffX*     xf;             // the classes' forbidden groups >= 64, packed (ClassAff.xf_off)
  const uint32_t* xc;             // the classes' joined groups >= 64, packed (ClassAff.xc_off)
  const int32_t*  w_kind;
  const int32_t*  w_keyset;
  const int64_t*  w_value;
  const uint8_t*  kind_unbound;   // [n_kinds]
  int32_t*   cnt;                 // mutable: group counters
  int32_t*   total;               // [n_groups]
  int32_t*   kind_count;          // [n_kinds][N]
  int32_t*   first_unbound;       // [1], -1 none
  long long* dom_sum;             // [dom_total] scratch of the priority: weight per domain over the feasible nodes (pass 1)
  long long* minmax;              // [3] min / max count over the feasible nodes (pass 2); [2] = max preferred node-affinity count
};

// Must the replay stop after ONE placement of this class (fresh scan per task)?  Yes when its keys read counters that its own
// placement changes beyond the chosen node: a weight list (allocate view: nodeorder on), or predicate groups over multi-node domains.
KB_HD bool aff_stop_each(const ClassAff& ca, const bool nodeorder) {
  if (ca.w_cnt != 0 && nodeorder) return true;
  if (ca.forbid == 0 && ca.xf_cnt == 0 && ca.need < 0) return false;
  return ca.pred_multi_ok == 0;
}

KB_HD uint32_t aff_lowest_bit(const uint64_t m) {
#if defined(__CUDA_ARCH__)
  return (uint32_t)__ffsll((long long)m) - 1u;
#else
  return (uint32_t)__builtin_ctzll(m);
#endif
}

// predicate step 10 for a pod of class `ca` on node n (the predicates plugin must be enabled; the caller checks).
// The counter reads of up to four groups are issued together: each is a chain node_domain -> cnt (an L2 round trip each), and a
// lone thread only overlaps what it has in flight at once (a class forbidden by 35 groups would cost 35 serial round trips).
// Groups >= 64 come from the class's forbidden list: its first `ns` entries from `xs` (the scan stages them in shared memory),
// the rest from A.xf.
KB_HD bool aff_pred(const AffDev& A, const ClassAff& ca, const uint32_t N, const uint32_t n, const AffX* xs = nullptr,
                    const uint32_t ns = 0) {
  bool ok = true;
  uint64_t f = ca.forbid;
  while (f) {                                    // satisfiesExistingPodsAntiAffinity (:1400-1439) + the pod's own anti-affinity (:1526-1533)
    int32_t d[4];
    uint32_t off[4];
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int k = 0; k < 4; ++k) {
      d[k] = -1; off[k] = 0;
      if (f) {
        const uint32_t g = aff_lowest_bit(f);
        f &= f - 1;
        d[k] = A.node_domain[(size_t)A.group_keyset[g] * N + n];
        off[k] = A.group_off[g];
      }
    }
    int32_t v[4];
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int k = 0; k < 4; ++k) v[k] = d[k] >= 0 ? KB_LDM(&A.cnt[off[k] + (uint32_t)d[k]]) : 0;
    ok = ok && ((v[0] | v[1] | v[2] | v[3]) <= 0);          // counters are never negative
  }
  for (uint32_t i = 0; A.has_x && i < ca.xf_cnt; i += 4) {   // the same for the groups >= 64
    int32_t d[4];
    uint32_t off[4];
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int k = 0; k < 4; ++k) {
      d[k] = -1; off[k] = 0;
      const uint32_t j = i + (uint32_t)k;
      if (j < ca.xf_cnt) {
        const AffX x = j < ns ? xs[j] : A.xf[ca.xf_off + j];
        d[k] = A.node_domain[(size_t)x.row + n];
        off[k] = x.off;
      }
    }
    int32_t v[4];
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int k = 0; k < 4; ++k) v[k] = d[k] >= 0 ? KB_LDM(&A.cnt[off[k] + (uint32_t)d[k]]) : 0;
    ok = ok && ((v[0] | v[1] | v[2] | v[3]) <= 0);
  }
  if (ca.need >= 0) {                            // the pod's required affinity terms (:1516-1560)
    const uint32_t g = (uint32_t)ca.need;
    const int32_t d = A.node_domain[(size_t)A.group_keyset[g] * N + n];
    const bool match = d >= 0 && KB_LDM(&A.cnt[A.group_off[g] + (uint32_t)d]) > 0;
    const bool first_of_series = KB_LDM(&A.total[g]) == 0 && ca.self_match;
    ok = ok && (match || first_of_series);
  }
  return ok;
}

// ClassAff.self_block: does an ALLOCATED pod of the class forbid node n for the next pod of the class?  Only through a group it both
// joins and is forbidden by, and only if the node has a domain under the group's key set (a node without the label is never matched).
KB_HD bool aff_self_blocks(const AffDev& A, const ClassAff& ca, const uint32_t N, const uint32_t n) {
  uint64_t m = ca.self_block ? (ca.contrib & ca.forbid) : 0ull;
  while (m) {
    const uint32_t g = aff_lowest_bit(m);
    m &= m - 1;
    if (A.node_domain[(size_t)A.group_keyset[g] * N + n] >= 0) return true;
  }
  const uint32_t xs = (A.has_x && ca.self_block) ? ca.xs_cnt : 0u;
  for (uint32_t i = 0; i < xs; ++i)
    if (A.node_domain[(size_t)A.xf[ca.xf_off + i].row + n] >= 0) return true;
  return false;
}

// priority pass 1, one FEASIBLE node m: the weight its pods contribute, added to the domain of the "pod's node" per key set.
// `add(slot, value)` accumulates into dom_sum (atomicAdd on the device).  (i0, stride): the device gives a node to a whole warp
// and lane l the entries l, l + 32, ... — a class can weigh hundreds of pod kinds, and each test is an L2 read.
template <class Add>
KB_HD void aff_pass1_node(const AffDev& A, const ClassAff& ca, const uint32_t N, const uint32_t m, Add add,
                          const uint32_t i0 = 0, const uint32_t stride = 1) {
  const int32_t fu = KB_LDM(A.first_unbound);
  for (uint32_t i = ca.w_off + i0; i < ca.w_off + ca.w_cnt; i += stride) {
    const uint32_t e = (uint32_t)A.w_kind[i], ks = (uint32_t)A.w_keyset[i];
    const int32_t c = KB_LDM(&A.kind_count[(size_t)e * N + m]);
    if (!c) continue;
    const uint32_t fixed = A.kind_unbound[e] ? (uint32_t)fu : m;     // cachedNodeInfo.GetNodeInfo (nodeorder.go:49-63)
    const int32_t d = A.node_domain[(size_t)ks * N + fixed];
    if (d >= 0) add(A.keyset_off[ks] + (uint32_t)d, (long long)A.w_value[i] * (long long)c);
  }
}
// pass 2 / 3, one feasible node n: pm.counts[n]
KB_HD long long aff_count_node(const AffDev& A, const ClassAff& ca, const uint32_t N, const uint32_t n) {
  long long count = 0;
  uint64_t k = ca.w_keysets;
  while (k) {
    const uint32_t ks = aff_lowest_bit(k);
    k &= k - 1;
    const int32_t d = A.node_domain[(size_t)ks * N + n];
    if (d >= 0) count += KB_LDM(&A.dom_sum[A.keyset_off[ks] + (uint32_t)d]);
  }
  return count;
}
// interpod_affinity.go:222-228: fScore = MaxPriority * (float64(count - min) / float64(max - min)); int(fScore); 0 if max == min
KB_HD int64_t aff_score(const long long count, const long long mn, const long long mx) {
  if (mx - mn <= 0) return 0;
  return (int64_t)KB_D2LL(KB_DMUL(10.0, KB_DDIV(KB_LL2D(count - mn), KB_LL2D(mx - mn))));
}
KB_HD uint64_t aff_add_score(const uint64_t key, const int32_t w_podaff, const int64_t score) {
  if (!key) return key;
  const int64_t hi = (int64_t)(key >> 32) + (int64_t)w_podaff * score;
  return ((uint64_t)hi << 32) | (key & 0xFFFFFFFFull);
}

// One placement of a task of class `ca` on node n (single thread): what ssn.Allocate / ssn.Pipeline change for the pods that
// come after it.
KB_HD void aff_commit(const AffDev& A, const ClassAff& ca, const uint32_t N, const uint32_t n, const bool allocated) {
  if (allocated) {
    uint64_t c = ca.contrib;
    while (c) {
      const uint32_t g = aff_lowest_bit(c);
      c &= c - 1;
      A.total[g] = KB_LDM(&A.total[g]) + 1;
      const int32_t d = A.node_domain[(size_t)A.group_keyset[g] * N + n];
      if (d >= 0) A.cnt[A.group_off[g] + (uint32_t)d] = KB_LDM(&A.cnt[A.group_off[g] + (uint32_t)d]) + 1;
    }
    for (uint32_t i = 0; A.has_x && i < ca.xc_cnt; ++i) {
      const uint32_t g = A.xc[ca.xc_off + i];
      A.total[g] = KB_LDM(&A.total[g]) + 1;
      const int32_t d = A.node_domain[(size_t)A.group_keyset[g] * N + n];
      if (d >= 0) A.cnt[A.group_off[g] + (uint32_t)d] = KB_LDM(&A.cnt[A.group_off[g] + (uint32_t)d]) + 1;
    }
  }
  if (ca.kind >= 0) A.kind_count[(size_t)ca.kind * N + n] = KB_LDM(&A.kind_count[(size_t)ca.kind * N + n]) + 1;
  const int32_t fu = KB_LDM(A.first_unbound);
  if (fu < 0 || (int32_t)n < fu) *A.first_unbound = (int32_t)n;
}
// Statement.unpipeline of such a task (node.RemoveTask): its kind count on n goes down again.  first_unbound is a min over the
// placed pods and cannot be undone here: the caller restores the value it saved when the Statement opened.
KB_HD void aff_unpipeline(const AffDev& A, const ClassAff& ca, const uint32_t N, const uint32_t n) {
  if (ca.kind >= 0) A.kind_count[(size_t)ca.kind * N + n] = KB_LDM(&A.kind_count[(size_t)ca.kind * N + n]) - 1;
}

}  // namespace kb
#endif  // KB_AFF_H_
