// kb_build.h — CUDA-free host-side construction of a session from the C-ABI snapshot:
// plugin resolution by name, task equivalence classes, TaskOrderFn order, TMA node tiles, drf /
// proportion OnSessionOpen precomputation, per-queue job lists, the queue heap and the first visit.
// Used by kb_engine.cu (which uploads the two slabs) and by tests/emu (which runs them on the CPU).
#ifndef KB_BUILD_H_
#define KB_BUILD_H_

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <type_traits>
#include <unordered_map>
#include <map>
#include <vector>

#include "kb_ctl.h"

namespace kb {

struct Slab {                       // bump allocator over one byte buffer; offsets are 256-byte aligned
  std::vector<unsigned char> host;  // sized (and zeroed) ONCE by commit(): the capacity is reused when the Slab is
  size_t top = 0;
  void reset() { top = 0; }
  size_t alloc(size_t bytes) {
    const size_t off = (top + 255) & ~(size_t)255;
    top = off + bytes;
    return off;
  }
  void commit() { host.assign((top + 255) & ~(size_t)255, 0); }
};

struct HostRes { double v[KB_MAX_R]; uint32_t present; HostRes() : present(0) { for (double& x : v) x = 0; } };

struct BuildErr { int code = 0; std::string msg; };
inline int bfail(BuildErr* e, int code, const char* fmt, ...) {
  char buf[512];
  va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
  e->code = code; e->msg = buf;
  return code;
}

inline bool parse_int(const char* s, int* out) {
  if (!s || !*s) return false;
  char* end = nullptr;
  long v = strtol(s, &end, 10);
  if (end == s || *end != '\0') return false;     // strconv.Atoi error: keep the default (arguments.go:36-43)
  *out = (int)v; return true;
}
inline bool parse_bool(const char* s, bool* out) {          // strconv.ParseBool (arguments.go:56-63)
  if (!s) return false;
  static const char* T[] = {"1", "t", "T", "TRUE", "true", "True"};
  static const char* F[] = {"0", "f", "F", "FALSE", "false", "False"};
  for (auto x : T) if (!strcmp(s, x)) { *out = true; return true; }
  for (auto x : F) if (!strcmp(s, x)) { *out = false; return true; }
  return false;
}

struct HostConf {
  EvalConf cf{};
  uint32_t jobcmp[4] = {0, 0, 0, 0};
  int w_nodeaff = 1;                // nodeaffinity.weight (nodeorder.go:111-117); only read when the session has preferred terms
  int w_podaff = 1;                 // podaffinity.weight; only read when the session carries kb_pod_affinity
  bool task_order_priority = false, queue_order_proportion = false, proportion_present = false, drf_present = false,
       gang_ready = false;
  // reclaim / preempt (kb_evict.h): EvictFn bits of the first tier with an enabled reclaimableFn / preemptableFn, and whether
  // gang's JobPipelinedFn is enabled
  uint32_t reclaim_fns = 0, preempt_fns = 0;
  bool gang_pipelined = false;
};

// plugins/factory.go:31-42 by name; OnSessionOpen registrations resolved in tier order (session_plugins.go)
inline int resolve_conf(BuildErr* e, const kb_plugin_conf* conf, uint32_t R, uint32_t W, HostConf& hc) {
  hc.cf.R = R; hc.cf.W = W;
  int w_least = 1, w_most = 0, w_nodeaff = 1, w_podaff = 1, w_bal = 1;      // nodeorder.go:111-117
  bool memp = false, diskp = false, pidp = false;                            // predicates.go:88-92
  bool have[7] = {false};
  enum { P_PRIORITY, P_GANG, P_DRF, P_PREDICATES, P_PROPORTION, P_NODEORDER, P_CONFORMANCE };
  static const char* names[] = {"priority", "gang", "drf", "predicates", "proportion", "nodeorder", "conformance"};
  auto id_of = [&](const char* n) { for (int i = 0; i < 7; ++i) if (n && !strcmp(n, names[i])) return i; return -1; };
  if (conf) {
    // pass 1: which plugins exist (every configured plugin's OnSessionOpen runs), arguments of the last occurrence win
    for (uint32_t t = 0; t < conf->n_tiers; ++t)
      for (uint32_t p = 0; p < conf->tiers[t].n_plugins; ++p) {
        const kb_plugin_option& o = conf->tiers[t].plugins[p];
        int id = id_of(o.name);
        if (id < 0) return bfail(e, KB_E_UNSUPPORTED_PLUGIN, "plugin '%s' is not a built-in: the GPU path honours built-in plugins by name only", o.name ? o.name : "(null)");
        have[id] = true;
        if (id == P_NODEORDER) { w_least = 1; w_most = 0; w_nodeaff = 1; w_podaff = 1; w_bal = 1; }
        if (id == P_PREDICATES) { memp = diskp = pidp = false; }
        for (uint32_t a = 0; a < o.n_args; ++a) {
          const char* k = o.arg_keys[a]; const char* v = o.arg_values[a];
          if (!k) continue;
          if (id == P_NODEORDER) {
            if (!strcmp(k, "leastrequested.weight")) parse_int(v, &w_least);
            else if (!strcmp(k, "mostrequested.weight")) parse_int(v, &w_most);
            else if (!strcmp(k, "nodeaffinity.weight")) parse_int(v, &w_nodeaff);
            else if (!strcmp(k, "podaffinity.weight")) parse_int(v, &w_podaff);
            else if (!strcmp(k, "balancedresource.weight")) parse_int(v, &w_bal);
          } else if (id == P_PREDICATES) {
            if (!strcmp(k, "predicate.MemoryPressureEnable")) parse_bool(v, &memp);
            else if (!strcmp(k, "predicate.DiskPressureEnable")) parse_bool(v, &diskp);
            else if (!strcmp(k, "predicate.PIDPressureEnable")) parse_bool(v, &pidp);
          }
        }
      }
    // pass 2: dispatch chains in tier / plugin order
    int nj = 0;
    auto in_chain = [&](uint32_t c) { for (int i = 0; i < nj; ++i) if (hc.jobcmp[i] == c) return true; return false; };
    for (uint32_t t = 0; t < conf->n_tiers; ++t) {
      // session_plugins.go:80-162: the first tier in which any enabled plugin registered a filter decides (an empty result
      // stays empty through the later tiers).  Registrations: gang.go:93-94, priority.go:100, drf.go:110, proportion.go:196,
      // conformance.go:61-62.  EvictFn bit values are spelled out here (kb_evict.h): gang 1, priority 2, drf 4, proportion 8, conformance 16.
      uint32_t rf = 0, pf = 0;
      for (uint32_t p = 0; p < conf->tiers[t].n_plugins; ++p) {
        const kb_plugin_option& o = conf->tiers[t].plugins[p];
        const int id = id_of(o.name);
        if (o.enabled_reclaimable) rf |= id == P_GANG ? 1u : id == P_PROPORTION ? 8u : id == P_CONFORMANCE ? 16u : 0u;
        if (o.enabled_preemptable) pf |= id == P_GANG ? 1u : id == P_PRIORITY ? 2u : id == P_DRF ? 4u : id == P_CONFORMANCE ? 16u : 0u;
        if (o.enabled_job_pipelined && id == P_GANG) hc.gang_pipelined = true;
      }
      if (!hc.reclaim_fns) hc.reclaim_fns = rf;
      if (!hc.preempt_fns) hc.preempt_fns = pf;
    }
    for (uint32_t t = 0; t < conf->n_tiers; ++t)
      for (uint32_t p = 0; p < conf->tiers[t].n_plugins; ++p) {
        const kb_plugin_option& o = conf->tiers[t].plugins[p];
        int id = id_of(o.name);
        if (o.enabled_job_order) {
          uint32_t c = id == P_PRIORITY ? JOBCMP_PRIORITY : id == P_GANG ? JOBCMP_GANG : id == P_DRF ? JOBCMP_DRF : JOBCMP_NONE;
          if (c != JOBCMP_NONE && !in_chain(c) && nj < 3) hc.jobcmp[nj++] = c;
        }
        if (o.enabled_task_order && id == P_PRIORITY) hc.task_order_priority = true;
        if (o.enabled_queue_order && id == P_PROPORTION) hc.queue_order_proportion = true;
        if (o.enabled_job_ready && id == P_GANG) hc.gang_ready = true;
        if (o.enabled_predicate && id == P_PREDICATES) hc.cf.predicates = 1;
        if (o.enabled_node_order && id == P_NODEORDER) hc.cf.nodeorder = 1;
      }
  }
  hc.proportion_present = have[P_PROPORTION];     // Overused ignores Enabled* (session_plugins.go:165-179)
  hc.drf_present = have[P_DRF];
  hc.cf.mem_pressure = memp; hc.cf.disk_pressure = diskp; hc.cf.pid_pressure = pidp;
  hc.cf.w_least = w_least; hc.cf.w_most = w_most; hc.cf.w_balanced = w_bal;
  hc.w_nodeaff = w_nodeaff;           // NodeAffinityPriority is identically 0 without preferred terms
  hc.w_podaff = w_podaff;             // InterPodAffinityPriority is identically 0 without inter-pod terms (kb_pod_affinity)
  const long lim = 1 << 20;
  if (labs(w_least) > lim || labs(w_most) > lim || labs(w_bal) > lim) return bfail(e, KB_E_BADARG, "nodeorder weight out of range");
  hc.cf.score_bias = 10ll * ((w_least < 0 ? -w_least : 0) + (w_most < 0 ? -w_most : 0) + (w_bal < 0 ? -w_bal : 0));
  return KB_OK;
}

// ---- host-side Resource algebra with scalar-map presence, for proportion's OnSessionOpen only ----
inline void hr_add(uint32_t R, HostRes& r, const HostRes& rr) {            // resource_info.go:128-140
  r.v[0] += rr.v[0]; r.v[1] += rr.v[1];
  for (uint32_t k = 2; k < R; ++k) if ((rr.present >> k) & 1u) { r.present |= 1u << k; r.v[k] += rr.v[k]; }
}
inline bool hr_le(uint32_t R, const HostRes& l, const HostRes& r) {        // :268-302
  return res_less_equal(R, [&](uint32_t k) { return ((k < 2) || ((l.present >> k) & 1u)) ? l.v[k] : 0.0; },
                        [&](uint32_t k) { return ((k < 2) || ((r.present >> k) & 1u)) ? r.v[k] : 0.0; });
}
inline bool hr_less(uint32_t R, const HostRes& r, const HostRes& rr) {     // :227-265
  if (!(r.v[0] < rr.v[0])) return false;
  if (!(r.v[1] < rr.v[1])) return false;
  if (r.present == 0) {
    if (rr.present != 0)
      for (uint32_t k = 2; k < R; ++k) if (((rr.present >> k) & 1u) && rr.v[k] <= KB_MIN_MILLI_SCALAR) return false;
    return true;
  }
  if (rr.present == 0) return false;
  for (uint32_t k = 2; k < R; ++k) {
    if (!((r.present >> k) & 1u)) continue;
    double q = ((rr.present >> k) & 1u) ? rr.v[k] : 0.0;
    if (!(r.v[k] < q)) return false;
  }
  return true;
}
inline HostRes hr_min(uint32_t R, const HostRes& l, const HostRes& r) {    // helpers.go:28-44
  HostRes res;
  res.v[0] = std::fmin(l.v[0], r.v[0]); res.v[1] = std::fmin(l.v[1], r.v[1]);
  if (l.present == 0 || r.present == 0) return res;
  for (uint32_t k = 2; k < R; ++k) if ((l.present >> k) & 1u) {
    res.present |= 1u << k;
    res.v[k] = std::fmin(l.v[k], ((r.present >> k) & 1u) ? r.v[k] : 0.0);
  }
  return res;
}
inline void hr_diff(uint32_t R, const HostRes& r, const HostRes& rr, HostRes& inc, HostRes& dec) {   // :305-337
  inc = HostRes(); dec = HostRes();
  for (uint32_t k = 0; k < 2; ++k) { if (r.v[k] > rr.v[k]) inc.v[k] += r.v[k] - rr.v[k]; else dec.v[k] += rr.v[k] - r.v[k]; }
  for (uint32_t k = 2; k < R; ++k) {
    if (!((r.present >> k) & 1u)) continue;
    double q = ((rr.present >> k) & 1u) ? rr.v[k] : 0.0;
    if (r.v[k] > q) { inc.present |= 1u << k; inc.v[k] += r.v[k] - q; }
    else { dec.present |= 1u << k; dec.v[k] += q - r.v[k]; }
  }
}
inline bool hr_sub(uint32_t R, HostRes& r, const HostRes& rr) {            // :143-160, false where the reference panics
  if (!hr_le(R, rr, r)) return false;
  r.v[0] -= rr.v[0]; r.v[1] -= rr.v[1];
  for (uint32_t k = 2; k < R; ++k) {
    if (!((rr.present >> k) & 1u)) continue;
    if (r.present == 0) return true;
    r.present |= 1u << k; r.v[k] -= rr.v[k];
  }
  return true;
}
inline bool hr_is_empty(uint32_t R, const HostRes& r) {                    // :93-105
  if (!(r.v[0] < KB_MIN_MILLI_CPU && r.v[1] < KB_MIN_MEMORY)) return false;
  for (uint32_t k = 2; k < R; ++k) if (((r.present >> k) & 1u) && r.v[k] >= KB_MIN_MILLI_SCALAR) return false;
  return true;
}



struct OffMut { size_t tiles, used, job_pos, job_ready, job_alloc, job_share, job_placed, q_head, dyn, q_dyn, q_alloc, q_share, qheap, dec, cand, ctl, sendbuf, recvbuf,
                bf_job_pos, bf_ctl, pipe_g, modlog, pcand, ppref, aff_cnt, aff_total, aff_kind_count, aff_first_unbound, aff_dom_sum, aff_minmax; };
struct OffImm { size_t classes, ord_task, ord_class, ord_run, ord_peek, job_ord_off, job_min, job_queue, job_prio, job_tb, q_static, q_static_off, q_des, q_des_p, q_ctime, task_class, job_ready0,
                bf_ord_task, bf_ord_class, bf_ord_run, bf_ord_peek, bf_job_ord_off, bf_jobs, bf_jobs_off, bf_classes, ord_chain, class_pref,
                aff_node_domain, aff_keyset_off, aff_group_keyset, aff_group_off, aff_cls, aff_w_kind, aff_w_keyset, aff_w_value, aff_kind_unbound,
                aff_xf, aff_xc, total_hi; };

struct BuiltSession {
  Slab mut, imm;
  OffMut om{};
  OffImm oi{};
  HostConf hc;
  uint32_t R = 0, W = 0, N = 0, T = 0, J = 0, Q = 0, C = 0, NT = 0, ncols = 0, To = 0, grid = 1;
  RecKind rec = RecKind::Own;        // the record type of the class tables and preferred terms: rec_kind(R, W)
  uint32_t total_dims_mask = 3;
  double total[KB_MAX_R] = {0};
  std::vector<int32_t> job_min_avail;
  uint32_t rank = 0, world = 1, tile_lo = 0, tile_hi = 0, nodes_per_rank = 0, tpi = 1, overlap = 0;
  uint32_t kchain = 1;               // classes per launch (visit_chain_kernel), 1 = off
  uint32_t pipe = 0, pipe_S = 0, pipe_tpc = 0;   // persistent pipeline (cycle_kernel): scanner CTAs, resident tiles per scanner CTA
  std::vector<ClassPref> class_pref; // [C] preferred node-affinity terms per class — HOST ONLY (read by tests/emu's prototype of
  bool has_pref = false;             // the two-pass scan); the device slabs do not carry them yet
  AffDev aff{};                      // inter-pod (anti)affinity: sizes and flags (pointers are set by bind())
  bool aff_session = false;          // the snapshot carries kb_pod_affinity (counter path OR atoms)
  bool aff_evict_ok = true;          // reclaim / preempt may run: no affinity tables, or host-level anti-affinity as atoms.  A victim that
                                     // is no member changes nothing, preemptors are Pipelined (never members); an evicted MEMBER clears its
                                     // atoms through the member counts of kb_evict_build.h, or withholds the outcome when kb_running carries
                                     // no group lists (KB_RUNNING_AFF_MEMBER).  On the counter path: no class reads a counter group in
                                     // predicate step 10 (aff_groups_unread); the evicting actions then keep kind_count / first_unbound
                                     // of InterPodAffinityPriority (kb_evict.h)
  bool aff_groups_unread = false;    // counter path, and no class has forbid / xf_cnt / need >= 0 with the predicates plugin on: a
                                     // member's eviction (it leaves util.PodLister) changes nothing any predicate reads
  uint64_t aff_atom_mask[KB_MAX_W] = {0};   // port-word bits that encode host-level anti-affinity groups (hidden from kb_node_state)
  std::vector<int32_t> aff_atom_of_group;   // [n_groups] group -> port-word bit of its atom, -1 (not an atom: nobody reads or joins it);
                                            // empty unless the session's groups became atoms
  uint32_t Tb = 0;                   // backfill order slots: Pending tasks with InitResreq.IsEmpty() (backfill.go:47)
  std::vector<uint32_t> q_alloc_present;   // [Q] scalar presence of proportion's queueAttr.allocated at session open (kb_evict.h: Resource.Less)

  // The BACKFILL VIEW of the same session (backfillAction.Execute, actions/backfill/backfill.go:40-71): same node table,
  // job / queue accounting, decisions and exchange buffers; its own task order (best-effort tasks only), cursors and
  // control block; no resource predicate, no nodeorder (the first node that passes wins = lowest node index).
  void bind_backfill(DevSession& D, unsigned char* mb, unsigned char* ib) const {
    bind(D, mb, ib);
    D.backfill = 1; D.overlap = 0; D.kchain = 1; D.pipe = 0;
    D.cf.fit_mode = hc.cf.predicates ? 2 : 1; D.cf.nodeorder = 0; D.cf.score_bias = 0;
    D.To = Tb;
    D.classes = (ClassRec*)(ib + oi.bf_classes);        // same ids; `initreq` holds Resreq (EvalConf.fit_mode)
    D.ord_task = (uint32_t*)(ib + oi.bf_ord_task); D.ord_class = (uint32_t*)(ib + oi.bf_ord_class);
    D.ord_run = (uint32_t*)(ib + oi.bf_ord_run); D.ord_peek = (uint32_t*)(ib + oi.bf_ord_peek);
    D.job_ord_off = (uint32_t*)(ib + oi.bf_job_ord_off);
    D.job_pos = (uint32_t*)(mb + om.bf_job_pos);
    D.q_static = (uint32_t*)(ib + oi.bf_jobs); D.q_static_off = (uint32_t*)(ib + oi.bf_jobs_off);
    D.ctl = (Ctl*)(mb + om.bf_ctl);
  }

  void bind(DevSession& D, unsigned char* mb, unsigned char* ib) const {
    D.cf = hc.cf;
    D.N = N; D.T = T; D.J = J; D.Q = Q; D.C = C; D.NT = NT; D.ncols = ncols; D.To = To;
    D.gang_ready = hc.gang_ready ? 1 : 0;
    for (int i = 0; i < 4; ++i) D.jobcmp[i] = hc.jobcmp[i];
    D.queue_order_proportion = hc.queue_order_proportion; D.proportion_present = hc.proportion_present; D.drf_present = hc.drf_present;
    D.total_dims_mask = total_dims_mask;
    for (uint32_t r = 0; r < KB_CLASS_R; ++r) D.total[r] = total[r];
    D.total_hi = (const double*)(ib + oi.total_hi);
    D.tiles = (uint64_t*)(mb + om.tiles); D.node_used = (double*)(mb + om.used);
    D.job_pos = (uint32_t*)(mb + om.job_pos); D.job_ready = (int32_t*)(mb + om.job_ready);
    D.job_alloc = (double*)(mb + om.job_alloc); D.job_share = (double*)(mb + om.job_share);
    D.job_placed = (uint32_t*)(mb + om.job_placed); D.q_static_head = (uint32_t*)(mb + om.q_head);
    D.dyn_jobs = (uint32_t*)(mb + om.dyn); D.q_dyn_len = (uint32_t*)(mb + om.q_dyn); D.q_allocated = (double*)(mb + om.q_alloc); D.q_share = (double*)(mb + om.q_share);
    D.qheap = (uint32_t*)(mb + om.qheap); D.dec = (kb_decision*)(mb + om.dec); D.cand = (uint64_t*)(mb + om.cand);
    D.ctl = (Ctl*)(mb + om.ctl);
    D.tpi = tpi;
    D.rank = rank; D.world = world; D.tile_lo = tile_lo; D.tile_hi = tile_hi; D.nodes_per_rank = nodes_per_rank;
    D.sendbuf = (uint64_t*)(mb + om.sendbuf); D.recvbuf = (uint64_t*)(mb + om.recvbuf);
    D.classes = (ClassRec*)(ib + oi.classes); D.ord_task = (uint32_t*)(ib + oi.ord_task); D.ord_class = (uint32_t*)(ib + oi.ord_class);
    D.ord_run = (uint32_t*)(ib + oi.ord_run); D.ord_peek = (uint32_t*)(ib + oi.ord_peek);
    D.overlap = overlap;
    D.kchain = kchain; D.ord_chain = (uint32_t*)(ib + oi.ord_chain);
    D.pipe = pipe; D.pipe_S = pipe_S; D.pipe_tpc = pipe_tpc; D.pipe_pad = 0;
    D.pg = (PipeG*)(mb + om.pipe_g); D.modlog = (uint32_t*)(mb + om.modlog); D.pcand = (uint64_t*)(mb + om.pcand);
    D.dbg = nullptr;
    D.ppref = (unsigned long long*)(mb + om.ppref);
    D.class_pref = has_pref ? (const ClassPref*)(ib + oi.class_pref) : nullptr;
    D.w_nodeaff = hc.w_nodeaff;
    D.aff = aff;
    if (aff.on) {
      D.aff.node_domain = (const int32_t*)(ib + oi.aff_node_domain); D.aff.keyset_off = (const uint32_t*)(ib + oi.aff_keyset_off);
      D.aff.group_keyset = (const uint32_t*)(ib + oi.aff_group_keyset); D.aff.group_off = (const uint32_t*)(ib + oi.aff_group_off);
      D.aff.cls = (const ClassAff*)(ib + oi.aff_cls);
      D.aff.xf = (const AffX*)(ib + oi.aff_xf); D.aff.xc = (const uint32_t*)(ib + oi.aff_xc);
      D.aff.w_kind = (const int32_t*)(ib + oi.aff_w_kind); D.aff.w_keyset = (const int32_t*)(ib + oi.aff_w_keyset);
      D.aff.w_value = (const int64_t*)(ib + oi.aff_w_value); D.aff.kind_unbound = (const uint8_t*)(ib + oi.aff_kind_unbound);
      D.aff.cnt = (int32_t*)(mb + om.aff_cnt); D.aff.total = (int32_t*)(mb + om.aff_total);
      D.aff.kind_count = (int32_t*)(mb + om.aff_kind_count); D.aff.first_unbound = (int32_t*)(mb + om.aff_first_unbound);
      D.aff.dom_sum = (long long*)(mb + om.aff_dom_sum); D.aff.minmax = (long long*)(mb + om.aff_minmax);
    }
    D.job_ord_off = (uint32_t*)(ib + oi.job_ord_off); D.job_min_avail = (int32_t*)(ib + oi.job_min);
    D.job_queue = (uint32_t*)(ib + oi.job_queue); D.job_prio = (int32_t*)(ib + oi.job_prio); D.job_tb_rank = (uint32_t*)(ib + oi.job_tb);
    D.q_static = (uint32_t*)(ib + oi.q_static); D.q_static_off = (uint32_t*)(ib + oi.q_static_off);
    D.q_deserved = (double*)(ib + oi.q_des); D.q_deserved_present = (uint32_t*)(ib + oi.q_des_p); D.q_ctime = (int64_t*)(ib + oi.q_ctime);
  }
};

// tests/emu's first a12 prototype (plain launches + a countdown of the feasible max-count nodes in the replay) only survives for the
// SHARDED emulation (world > 1: pass 1 on every rank's replicated table, no second exchange); on one rank the plain path now
// evaluates preferred node affinity like the kernels do (counter path)
inline bool allow_pref_legacy(bool allow_pref, uint32_t world) { return allow_pref && world > 1; }

// Tiles per scan iteration of the per-visit kernels: up to 4 (16 warps), bounded by the shared memory left for the two staging
// buffers next to VisitSmem — ~190 KB next to the narrow instances' ~26 KB, ~160 KB next to the wide instances' ~51 KB (class
// record and candidate slots of up to 82 columns) and the wide-atom instances' (up to 70 columns).  The widest records (R = 32,
// W = 4: 82 columns, 84 KB per tile; R = 8, W = 16: 70 columns, 72 KB per tile) get tpi = 1.
inline uint32_t scan_tpi(const uint32_t R, const uint32_t W) {
  const size_t tile_bytes = (size_t)tile_ncols(R, W) * TILE_NODES * 8;
  const size_t budget = (R > KB_NARROW_R || W > KB_NARROW_W ? 160 : 190) * 1024;
  uint32_t tpi = 4;
  while (tpi > 1 && 2 * tpi * tile_bytes > budget) --tpi;
  return tpi;
}

// Everything kb_session_load does before touching the device.  `max_grid` = scan CTAs (SM count).
inline int build_session(const kb_snapshot* s, const kb_plugin_conf* conf, uint32_t max_grid, BuiltSession& B, BuildErr* e,
                         uint32_t rank = 0, uint32_t world = 1, int overlap_mode = -1 /* -1 auto, 0 off, 1 on */,
                         uint32_t kchain = 1 /* classes per launch: 1, 2 or 4 (single GPU, no overlap) */,
                         bool allow_pref = false /* accept preferred node-affinity terms (tests/emu prototype only) */,
                         int pipe_mode = 0 /* persistent pipeline (cycle_kernel): 0 off, 1 when the geometry allows it */,
                         bool wide_classes = false /* the caller reads class tables of ClassRecWide / ClassRecAtoms (class_table<CR>):
                                                      sessions with R > KB_CLASS_R or W > KB_CLASS_W are accepted (the engine's wide and
                                                      wide-atom kernel instances) */) {
  if (!s) return bfail(e, KB_E_BADARG, "snapshot is NULL");
  if (s->abi_version != KB_ABI_VERSION) return bfail(e, KB_E_BADARG, "snapshot abi_version %u != %u", s->abi_version, KB_ABI_VERSION);
  const kb_pod_affinity* pa = s->pod_affinity;
  if ((s->flags & KB_SNAPSHOT_PLACED_POD_AFFINITY) && !pa)
    return bfail(e, KB_E_UNSUPPORTED_FEATURE, "a placed pod carries inter-pod (anti)affinity terms: the reference lets it reject nodes for other pods "
                 "(predicates.go:1261-1288); the flattener must hand over kb_snapshot.pod_affinity (no CPU fallback)");
  if (pa && pa->n_groups > KB_MAX_AFF_GROUPS)
    return bfail(e, KB_E_UNSUPPORTED_FEATURE, "kb_pod_affinity: %u counter groups, more than %u", pa->n_groups, (unsigned)KB_MAX_AFF_GROUPS);
  if (pa && pa->n_keysets > 64) return bfail(e, KB_E_UNSUPPORTED_FEATURE, "kb_pod_affinity: more than 64 key sets");
  if (s->flags & ~(KB_SNAPSHOT_PLACED_POD_AFFINITY | KB_SNAPSHOT_LISTED_POD_WITHOUT_NODE)) return bfail(e, KB_E_BADARG, "unknown kb_snapshot.flags bits 0x%x", s->flags);
  if (s->R < 2 || s->R > KB_MAX_R || s->W < 1 || s->W > KB_MAX_W)
    return bfail(e, KB_E_BADARG, "R=%u / W=%u out of range (2 <= R <= KB_MAX_R = %u, 1 <= W <= KB_MAX_W = %u)", s->R, s->W, (unsigned)KB_MAX_R, (unsigned)KB_MAX_W);
  // no record holds both: the widest node tile (R = 32, W = 16: 118 columns) would not fit next to the wide VisitSmem staging
  if (s->R > KB_NARROW_R && s->W > KB_NARROW_W)
    return bfail(e, KB_E_UNSUPPORTED_FEATURE, "R=%u resource dimensions with W=%u mask words: sessions with R > KB_NARROW_R (%u) take at most "
                 "KB_NARROW_W (%u) words, sessions with W > KB_NARROW_W at most KB_NARROW_R dimensions", s->R, s->W, (unsigned)KB_NARROW_R,
                 (unsigned)KB_NARROW_W);
  if (s->R > KB_CLASS_R && !wide_classes)
    return bfail(e, KB_E_BADARG, "R=%u: this build reads class records of %u resource dimensions (ClassRec)", s->R, (unsigned)KB_CLASS_R);
  if (s->W > KB_CLASS_W && !wide_classes)
    return bfail(e, KB_E_BADARG, "W=%u: this build reads class records of %u mask words (ClassRec)", s->W, (unsigned)KB_CLASS_W);
  // the sharded exchange carries node records of at most KB_NARROW_R dimensions and KB_NARROW_W words (P2P_RANK_U64)
  if (world > 1 && s->R > KB_NARROW_R)
    return bfail(e, KB_E_UNSUPPORTED_FEATURE, "R=%u resource dimensions with a sharded node axis (KB_ENGINE_SHARD): the exchange carries node records "
                 "of at most %u dimensions", s->R, (unsigned)KB_NARROW_R);
  if (world > 1 && s->W > KB_NARROW_W)
    return bfail(e, KB_E_UNSUPPORTED_FEATURE, "W=%u mask words with a sharded node axis (KB_ENGINE_SHARD): the exchange carries node records "
                 "of at most KB_NARROW_W (%u) words", s->W, (unsigned)KB_NARROW_W);
  if (s->Q > KB_MAX_Q) return bfail(e, KB_E_BADARG, "Q=%u > KB_MAX_Q (%u)", s->Q, (unsigned)KB_MAX_Q);
  if (s->N >= 0xFFFFFFF0u) return bfail(e, KB_E_BADARG, "N too large for the packed key");
  const uint32_t R = s->R, W = s->W, N = s->N, T = s->T, J = s->J, Q = s->Q;
  B.hc = HostConf();                 // a BuiltSession may be reused across loads (the engine keeps one to recycle its buffers)
  HostConf& hc = B.hc;
  int rc = resolve_conf(e, conf, R, W, hc);
  if (rc) return rc;
  B.aff_session = pa != nullptr;
  B.aff_evict_ok = pa == nullptr;
  B.aff_groups_unread = false;
  for (uint32_t w = 0; w < KB_MAX_W; ++w) B.aff_atom_mask[w] = 0;
  // Host-level inter-pod anti-affinity as ATOMS.  When every counter the session's tasks read or join lives on a key set whose
  // domains are exactly the nodes (kubernetes.io/hostname), "a member of group g sits in the node's domain" is a per-node bit,
  // set by an Allocate of a contributing task and tested like a host-port conflict (predicates.go:1153-1173 has the same shape):
  // group g becomes a spare bit of the port words, ClassRec.port_conflict gets the forbidden groups, ClassRec.aff_own the joined
  // ones (applied by Allocate only: a Pipelined pod is not listed by util.PodLister).  The placement then changes ONE node record
  // again, every invariant of the candidate lists holds (DESIGN.md 2) and the session runs on the persistent pipeline at full
  // speed.  Not convertible (-> per-visit kernels with counters, kb_aff.h): required pod AFFINITY, live priority weights, multi-node
  // domains, nodes without the topology label, no spare bits.  KB_AFF_ATOMS=0 forces the counter path.
  std::vector<int32_t>& aff_atom_of_group = B.aff_atom_of_group;   // group -> atom index, -1
  aff_atom_of_group.clear();
  std::vector<uint64_t> node_aff_bits;                  // [W][N] initial member bits
  std::vector<uint32_t> aff_group_off0;
  bool aff_as_atoms = false;
  // groups >= 64 of task t: the entries task_xgroup[xg_lo(t) .. xg_hi(t)), (g << 2) | KB_XGROUP_FORBID | KB_XGROUP_CONTRIB
  const uint32_t* xg_off = pa ? pa->task_xgroup_off : nullptr;
  const uint32_t* xg_ent = pa ? pa->task_xgroup : nullptr;
  auto xg_at = [&](uint32_t t, uint32_t i) { return xg_ent[xg_off[t] + i]; };
  auto xg_lo = [&](uint32_t t) { return xg_off ? xg_off[t] : 0u; };
  auto xg_hi = [&](uint32_t t) { return xg_off ? xg_off[t + 1] : 0u; };
  auto xg_same = [&](uint32_t t, uint32_t u) {       // tasks t and u name the same groups >= 64 in the same order
    if (xg_hi(t) - xg_lo(t) != xg_hi(u) - xg_lo(u)) return false;
    for (uint32_t i = 0; i < xg_hi(t) - xg_lo(t); ++i) if (xg_at(t, i) != xg_at(u, i)) return false;
    return true;
  };
  if (pa) {
    aff_group_off0.assign(pa->n_groups + 1, 0);
    uint64_t off = 0;
    for (uint32_t g = 0; g < pa->n_groups; ++g) {
      if (pa->group_keyset[g] >= pa->n_keysets) return bfail(e, KB_E_BADARG, "kb_pod_affinity: group %u names a key set out of range", g);
      off += pa->keyset_domains[pa->group_keyset[g]];
      if (off > 0xFFFFFFFFull) return bfail(e, KB_E_UNSUPPORTED_FEATURE, "kb_pod_affinity: the counters of %u groups do not fit 32-bit offsets", pa->n_groups);
      aff_group_off0[g + 1] = (uint32_t)off;
    }
    if (pa->n_groups > 64 && (uint64_t)pa->n_keysets * N > 0xFFFFFFFFull)
      return bfail(e, KB_E_UNSUPPORTED_FEATURE, "kb_pod_affinity: %u key sets x %u nodes do not fit 32-bit offsets", pa->n_keysets, N);
    if (xg_off) {
      for (uint32_t t = 0; t < T; ++t)
        if (xg_off[t] > xg_off[t + 1]) return bfail(e, KB_E_BADARG, "kb_pod_affinity: task_xgroup_off is not monotone at task %u", t);
      if (T && xg_off[T] > xg_off[0] && !pa->task_xgroup) return bfail(e, KB_E_BADARG, "kb_pod_affinity: task_xgroup is NULL but task_xgroup_off names entries");
      for (uint32_t i = T ? xg_off[0] : 0u; T && i < xg_off[T]; ++i) {
        const uint32_t x = pa->task_xgroup[i], g = x >> 2;
        if (g < 64 || g >= pa->n_groups || (x & 3u) == 0)
          return bfail(e, KB_E_BADARG, "kb_pod_affinity: task_xgroup entry %u (group %u, flags %u) is not a group >= 64 of the session", i, g, x & 3u);
      }
    }
    const char* sw = getenv("KB_AFF_ATOMS");
    bool ok = !(sw && atoi(sw) == 0);
    const bool weights_live = hc.cf.nodeorder && hc.w_podaff != 0;
    uint64_t used_lo = 0;                               // groups < 64 ...
    std::vector<uint8_t> used(pa->n_groups, 0);         // ... and every group a task reads or joins
    for (uint32_t t = 0; t < T && ok; ++t) {
      if (hc.cf.predicates && pa->task_need[t] >= 0) ok = false;
      if (weights_live && pa->task_weight_off[t + 1] > pa->task_weight_off[t]) ok = false;
      used_lo |= pa->task_contrib[t] | pa->task_forbid[t];
      for (uint32_t i = xg_lo(t); i < xg_hi(t); ++i) used[xg_ent[i] >> 2] = 1;
    }
    if (pa->n_groups < 64 && (used_lo >> pa->n_groups)) return bfail(e, KB_E_BADARG, "kb_pod_affinity: a task names a group out of range");
    for (uint32_t g = 0; g < pa->n_groups && g < 64; ++g) used[g] = (uint8_t)((used_lo >> g) & 1ull);
    if (!hc.cf.predicates) std::fill(used.begin(), used.end(), 0);    // step 10 is not evaluated: nothing reads the counters
    uint32_t n_used = 0;
    for (uint32_t g = 0; g < pa->n_groups; ++g) n_used += used[g];
    for (uint32_t g = 0; g < pa->n_groups && ok; ++g) {
      if (!used[g]) continue;
      const uint32_t ks = pa->group_keyset[g];
      if (pa->keyset_domains[ks] != N) { ok = false; break; }
      std::vector<uint8_t> seen(N, 0);
      for (uint32_t n = 0; n < N; ++n) {
        const int32_t d = pa->node_domain[(size_t)ks * N + n];
        if (d < 0 || d >= (int32_t)N || seen[d]) { ok = false; break; }
        seen[d] = 1;
      }
    }
    int hb = -1;                                        // highest port atom in use
    if (ok && n_used) {
      for (uint32_t w = 0; w < W; ++w) {
        uint64_t acc = 0;
        for (uint32_t n = 0; n < N; ++n) acc |= s->node_ports[(size_t)w * N + n];
        for (uint32_t t = 0; t < T; ++t) acc |= s->task_port_own[(size_t)w * T + t] | s->task_port_conflict[(size_t)w * T + t];
        if (acc) hb = (int)(w * 64 + 63 - (uint32_t)__builtin_clzll(acc));
      }
      if ((uint32_t)(hb + 1) + n_used > 64u * W) ok = false;
    }
    if (ok) {
      aff_as_atoms = true;
      aff_atom_of_group.assign(pa->n_groups, -1);
      node_aff_bits.assign((size_t)W * std::max(1u, N), 0);
      int next = hb + 1;
      for (uint32_t g = 0; g < pa->n_groups; ++g) {
        if (!used[g]) continue;
        const int a = next++;
        aff_atom_of_group[g] = a;
        B.aff_atom_mask[a / 64] |= 1ull << (a % 64);
        const uint32_t ks = pa->group_keyset[g];
        for (uint32_t n = 0; n < N; ++n)
          if (pa->group_count0[aff_group_off0[g] + (uint32_t)pa->node_domain[(size_t)ks * N + n]] > 0) node_aff_bits[(size_t)(a / 64) * N + n] |= 1ull << (a % 64);
      }
      B.aff_evict_ok = true;
    } else {
      // the counters of a topology domain change the keys of many nodes at once: per-visit kernels, fresh scan per task for
      // the classes that read them (kb_aff.h); no look-ahead lists, no overlap, no node sharding
      if (world > 1) return bfail(e, KB_E_UNSUPPORTED_FEATURE, "inter-pod affinity beyond host-level anti-affinity: not with a sharded node axis (KB_ENGINE_SHARD)");
      pipe_mode = 0; overlap_mode = 0; kchain = 1;
    }
  }
  const kb_pod_affinity* pa_full = pa;                  // the snapshot's tables (class identity below)
  if (aff_as_atoms) pa = nullptr;                       // from here on `pa` = what the counter path (AffDev) consumes
  // Preferred NODE affinity (a12) outside cycle_kernel: the per-visit kernels evaluate it with the same machinery as the inter-pod
  // priority — a pass over the feasible nodes before the visit (max count, aff_prepass_kernel<2>), the term in the scan, a fresh
  // scan per task of such a class.  Without inter-pod tables the counter path runs on empty ones.
  bool any_pref = false;
  for (uint32_t t = 0; t < T && !any_pref; ++t) any_pref = (s->task_flags[t] & KB_TASK_HAS_PREFERRED_NODE_AFFINITY) != 0;
  bool will_pipe = false;
  if (pipe_mode > 0 && world <= 1 && N > 0 && R == 3 && W == 2 && std::max(1u, max_grid) >= 2) {
    const uint32_t nt = (N + TILE_NODES - 1) / TILE_NODES, smax = std::max(1u, max_grid) - 1;
    const size_t tile_bytes = (size_t)tile_ncols(R, W) * TILE_NODES * 8;
    will_pipe = (nt + smax - 1) / smax <= (uint32_t)((227 * 1024 - 8 * 1024) / tile_bytes);
  }
  static const int32_t kz32[2] = {-1, -1};
  static const uint32_t kzu32[2] = {0, 0};
  static const uint64_t kzu64[2] = {0, 0};
  static const int64_t kz64[2] = {0, 0};
  static const uint8_t kzu8[2] = {0, 0};
  std::vector<uint64_t> empty_u64;
  std::vector<int32_t> empty_i32;
  std::vector<uint32_t> empty_off;
  kb_pod_affinity empty_pa;
  const bool pref_legacy = any_pref && allow_pref_legacy(allow_pref, world);
  const bool pref_on_counters = any_pref && !will_pipe && !pref_legacy;
  if (pref_on_counters || (pa && any_pref)) {
    if (world > 1) return bfail(e, KB_E_UNSUPPORTED_FEATURE, "preferred node-affinity terms outside the persistent pipeline: not with a sharded node axis");
    pipe_mode = 0; overlap_mode = 0; kchain = 1;
    if (!pa) {
      memset(&empty_pa, 0, sizeof empty_pa);
      empty_u64.assign(std::max(1u, T), 0); empty_i32.assign(std::max(1u, T), -1); empty_off.assign((size_t)T + 1, 0);
      empty_pa.first_unbound_node = -1;
      empty_pa.node_domain = kz32; empty_pa.keyset_domains = kzu32; empty_pa.group_keyset = kzu32; empty_pa.group_count0 = kz32 + 0;
      empty_pa.group_total0 = kz32; empty_pa.task_forbid = empty_u64.data(); empty_pa.task_need = empty_i32.data();
      empty_pa.task_contrib = empty_u64.data(); empty_pa.task_kind = empty_i32.data(); empty_pa.node_kind_count0 = kz32;
      empty_pa.kind_unbound = kzu8; empty_pa.task_weight_off = empty_off.data(); empty_pa.weight_kind = kz32; empty_pa.weight_keyset = kz32;
      empty_pa.weight_value = kz64;
      (void)kzu64;
      pa = &empty_pa;
    }
  }
  // the atoms of the groups task t forbids (flag KB_XGROUP_FORBID, mask task_forbid) or joins (KB_XGROUP_CONTRIB, task_contrib)
  auto atoms_of = [&](uint64_t groups, uint32_t t, uint32_t flag, uint64_t* out) {
    auto put = [&](uint32_t g) { const int a = aff_atom_of_group[g]; if (a >= 0) out[a / 64] |= 1ull << (a % 64); };
    while (groups) { const uint32_t g = (uint32_t)__builtin_ctzll(groups); groups &= groups - 1; put(g); }
    for (uint32_t i = xg_lo(t); i < xg_hi(t); ++i) if (xg_ent[i] & flag) put(xg_ent[i] >> 2);
  };

  // ---------------- validate + task classes ----------------
  for (uint32_t j = 0; j < J; ++j) {
    if (s->job_task_off[j] > s->job_task_off[j + 1] || s->job_task_off[j + 1] > T) return bfail(e, KB_E_BADARG, "job_task_off is not monotone at job %u", j);
    if (s->job_queue[j] >= Q) return bfail(e, KB_E_BADARG, "job %u: queue %u does not exist (cache.Snapshot drops such jobs, cache.go:652-656)", j, s->job_queue[j]);
  }
  if (J && (s->job_task_off[0] != 0 || s->job_task_off[J] != T)) return bfail(e, KB_E_BADARG, "job_task_off must cover [0,T)");
  // The reference's cache never hands out an over-committed node: node.AddTask refuses a task that does not fit into Idle
  // (api/node_info.go:161-167), so Idle >= -epsilon.  Outside that domain ssn.Allocate's "status first, node second" order
  // (framework/session.go:235-262) becomes observable, which this engine does not model.
  for (uint32_t n = 0; n < N; ++n)
    for (uint32_t r = 0; r < R; ++r) {
      const double eps = r == 0 ? KB_MIN_MILLI_CPU : r == 1 ? KB_MIN_MEMORY : KB_MIN_MILLI_SCALAR;
      if (s->node_idle[(size_t)r * N + n] <= -eps)
        return bfail(e, KB_E_BADARG, "node %u: Idle is negative in dim %u (over-committed node: the reference cache would not produce it)", n, r);
    }
  // the class identity: every dimension ClassRec holds and every mask word the session has; written to the class table in the
  // session's record type (write_classes)
  std::vector<ClassRecBuild> classes;
  // dims KB_CLASS_R..R-1 of every class (initreq, then resreq; empty when R <= KB_CLASS_R): part of the class identity, joined
  // with `classes` into the wide records of the class table
  const uint32_t RH = R > KB_CLASS_R ? R - KB_CLASS_R : 0u;
  std::vector<double> class_hi;
  std::vector<double> hi(2 * (size_t)RH, 0.0);
  auto init_of = [&](uint32_t id, uint32_t k) { return k < KB_CLASS_R ? classes[id].initreq[k] : class_hi[(size_t)id * 2 * RH + (k - KB_CLASS_R)]; };
  auto same_hi = [&](uint32_t id) { return RH == 0 || memcmp(&class_hi[(size_t)id * 2 * RH], hi.data(), 2 * (size_t)RH * 8) == 0; };
  std::vector<ClassPrefBuild> class_pref;
  B.class_pref.clear(); B.has_pref = false;
  auto pref_of = [&](uint32_t t) {
    ClassPrefBuild cp;
    memset(&cp, 0, sizeof cp);
    if (!(s->task_flags[t] & KB_TASK_HAS_PREFERRED_NODE_AFFINITY)) return cp;
    if (!s->task_n_pref_terms || !s->task_pref_terms || !s->task_pref_weights) { cp.n = 0xFFFFFFFFu; return cp; }   // reported by the caller
    cp.n = s->task_n_pref_terms[t];
    for (uint32_t p = 0; p < cp.n && p < KB_MAX_PREF_TERMS; ++p) {
      cp.weight[p] = s->task_pref_weights[(size_t)p * T + t];
      for (uint32_t w = 0; w < W; ++w) cp.term[p][w] = s->task_pref_terms[((size_t)p * W + w) * T + t];
    }
    return cp;
  };
  // inter-pod affinity: tasks with the same masks / kind / weight list share an "aff id", which is part of the class identity
  std::vector<uint32_t> aff_id(pa ? T : 0, 0);
  std::vector<ClassAff> aff_tab;                  // by aff id; w_off / w_cnt, xf_off / xc_off index the packed lists below
  std::vector<int32_t> aff_wk, aff_wks; std::vector<int64_t> aff_wv;
  std::vector<AffX> aff_xf; std::vector<uint32_t> aff_xc;
  std::vector<uint32_t> aff_xf_group;             // host only: the group of every aff_xf entry
  if (pa) {
    std::map<std::vector<int64_t>, uint32_t> ids;
    const bool xg_tab = pa == pa_full;            // not the empty tables of a session whose groups became atoms
    for (uint32_t t = 0; t < T; ++t) {
      std::vector<int64_t> key = {(int64_t)pa->task_forbid[t], (int64_t)pa->task_contrib[t], (int64_t)pa->task_need[t], (int64_t)pa->task_kind[t],
                                  (int64_t)((s->task_flags[t] & KB_TASK_AFF_SELF_MATCH) ? 1 : 0)};
      const uint32_t w0 = pa->task_weight_off[t], w1 = pa->task_weight_off[t + 1];
      if (w1 < w0 || w1 > pa->n_weights) return bfail(e, KB_E_BADARG, "kb_pod_affinity: task_weight_off is not monotone at task %u", t);
      for (uint32_t i = w0; i < w1; ++i) { key.push_back(pa->weight_kind[i]); key.push_back(pa->weight_keyset[i]); key.push_back(pa->weight_value[i]); }
      // groups >= 64 belong to the identity too (after the weights, with their count in front: no key of a smaller session changes)
      if (xg_tab && xg_hi(t) > xg_lo(t)) {
        std::vector<int64_t> xs;
        for (uint32_t i = xg_lo(t); i < xg_hi(t); ++i) xs.push_back(xg_ent[i]);
        std::sort(xs.begin(), xs.end());
        key.push_back(-(int64_t)xs.size() - 1);
        key.insert(key.end(), xs.begin(), xs.end());
      }
      auto it = ids.find(key);
      if (it == ids.end()) {
        if (pa->task_need[t] >= (int32_t)pa->n_groups || pa->task_kind[t] >= (int32_t)pa->n_kinds) return bfail(e, KB_E_BADARG, "kb_pod_affinity: task %u names a group / kind out of range", t);
        if (pa->n_groups < 64 && ((pa->task_forbid[t] | pa->task_contrib[t]) >> pa->n_groups)) return bfail(e, KB_E_BADARG, "kb_pod_affinity: task %u names a group out of range", t);
        ClassAff ca; memset(&ca, 0, sizeof ca);
        ca.forbid = pa->task_forbid[t]; ca.contrib = pa->task_contrib[t]; ca.need = pa->task_need[t]; ca.kind = pa->task_kind[t];
        ca.self_match = (s->task_flags[t] & KB_TASK_AFF_SELF_MATCH) ? 1u : 0u;
        ca.w_off = (uint32_t)aff_wk.size(); ca.w_cnt = w1 - w0;
        for (uint32_t i = w0; i < w1; ++i) {
          if (pa->weight_kind[i] < 0 || pa->weight_kind[i] >= (int32_t)pa->n_kinds || pa->weight_keyset[i] < 0 || pa->weight_keyset[i] >= (int32_t)pa->n_keysets)
            return bfail(e, KB_E_BADARG, "kb_pod_affinity: weight entry %u names a kind / key set out of range", i);
          aff_wk.push_back(pa->weight_kind[i]); aff_wks.push_back(pa->weight_keyset[i]); aff_wv.push_back(pa->weight_value[i]);
          ca.w_keysets |= 1ull << pa->weight_keyset[i];
        }
        if (xg_tab && xg_hi(t) > xg_lo(t)) {
          // forbidden groups >= 64, those the class also joins first (aff_self_blocks reads them), each resolved to (row, counters)
          std::vector<uint32_t> both, fonly, joined;
          for (uint32_t i = xg_lo(t); i < xg_hi(t); ++i) {
            const uint32_t x = xg_ent[i], g = x >> 2;
            if ((x & KB_XGROUP_FORBID) && (x & KB_XGROUP_CONTRIB)) both.push_back(g);
            else if (x & KB_XGROUP_FORBID) fonly.push_back(g);
            if (x & KB_XGROUP_CONTRIB) joined.push_back(g);
          }
          for (auto* v : {&both, &fonly, &joined}) { std::sort(v->begin(), v->end()); v->erase(std::unique(v->begin(), v->end()), v->end()); }
          fonly.erase(std::remove_if(fonly.begin(), fonly.end(), [&](uint32_t g) { return std::binary_search(both.begin(), both.end(), g); }), fonly.end());
          ca.xf_off = (uint32_t)aff_xf.size(); ca.xs_cnt = (uint32_t)both.size(); ca.xf_cnt = (uint32_t)(both.size() + fonly.size());
          for (auto* v : {&both, &fonly})
            for (const uint32_t g : *v) { aff_xf.push_back(AffX{pa->group_keyset[g] * N, aff_group_off0[g]}); aff_xf_group.push_back(g); }
          ca.xc_off = (uint32_t)aff_xc.size(); ca.xc_cnt = (uint32_t)joined.size();
          aff_xc.insert(aff_xc.end(), joined.begin(), joined.end());
        }
        it = ids.emplace(key, (uint32_t)aff_tab.size()).first;
        aff_tab.push_back(ca);
      }
      aff_id[t] = it->second;
    }
    if (aff_tab.size() >= (1u << 24)) return bfail(e, KB_E_UNSUPPORTED_FEATURE, "kb_pod_affinity: too many distinct affinity signatures");
    // Counter path: reclaim / preempt run when no class reads a counter group in predicate step 10.  The victim walk does not
    // follow the groups (an evicted member leaves util.PodLister), but then nothing reads them; InterPodAffinityPriority reads
    // NodeInfo.Tasks, which keeps an evicted pod as Releasing, and the evicting actions keep its kind counts (kb_evict.h).
    if (pa == pa_full && !aff_as_atoms) {
      bool reads = false;
      if (hc.cf.predicates)
        for (const ClassAff& ca : aff_tab) reads = reads || ca.forbid != 0 || ca.xf_cnt != 0 || ca.need >= 0;
      B.aff_groups_unread = !reads;
      B.aff_evict_ok = !reads;
    }
  }
  std::vector<uint32_t> task_class(T, 0);
  std::vector<uint8_t> task_empty(T, 0);
  {
    // open-addressing table keyed by a 64-bit hash of the record, verified field by field; a task usually equals its
    // predecessor (PodGroups are homogeneous), so that case is checked first.  Records and preferred terms are read through
    // their first W mask words only (the rest are 0), so a narrow session hashes and compares no more than its ClassRec.
    std::vector<uint32_t> table(1024, 0xFFFFFFFFu);
    std::vector<uint64_t> class_hash;
    auto rec_words = [W](const ClassRecBuild& c, auto&& fn) {
      for (uint32_t k = 0; k < KB_CLASS_R; ++k) { uint64_t a, b; memcpy(&a, &c.initreq[k], 8); memcpy(&b, &c.resreq[k], 8); fn(a); fn(b); }
      fn((uint64_t)c.nz_cpu); fn((uint64_t)c.nz_mem);
      for (uint32_t w = 0; w < W; ++w) {
        fn(c.sel_req[w]); fn(c.tol[w]); fn(c.port_own[w]); fn(c.port_conflict[w]); fn(c.aff_own[w]);
        for (uint32_t a = 0; a < KB_MAX_AFF_TERMS; ++a) fn(c.aff[a][w]);
      }
      fn(((uint64_t)c.n_aff << 32) | c.flags);
    };
    auto pref_words = [W](const ClassPrefBuild& p, auto&& fn) {
      for (uint32_t k = 0; k < KB_MAX_PREF_TERMS; ++k) {
        for (uint32_t w = 0; w < W; ++w) fn(p.term[k][w]);
        fn((uint64_t)(uint32_t)p.weight[k]);
      }
      fn(p.n);
    };
    auto hash_rec = [&](const ClassRecBuild& c) {
      uint64_t h = 0x9E3779B97F4A7C15ull;
      rec_words(c, [&](uint64_t x) { h ^= x + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2); h *= 0xFF51AFD7ED558CCDull; h ^= h >> 32; });
      return h;
    };
    auto same_rec = [&](const ClassRecBuild& a, const ClassRecBuild& b) {
      uint64_t va[KB_CLASS_R * 2 + 3 + 9 * KB_MAX_W];
      size_t n = 0, i = 0;
      bool same = true;
      rec_words(a, [&](uint64_t x) { va[n++] = x; });
      rec_words(b, [&](uint64_t x) { same = same && va[i++] == x; });
      return same;
    };
    auto same_pref = [&](const ClassPrefBuild& a, const ClassPrefBuild& b) {
      uint64_t va[KB_MAX_PREF_TERMS * (KB_MAX_W + 1) + 1];
      size_t n = 0, i = 0;
      bool same = true;
      pref_words(a, [&](uint64_t x) { va[n++] = x; });
      pref_words(b, [&](uint64_t x) { same = same && va[i++] == x; });
      return same;
    };
    uint32_t prev_class = 0xFFFFFFFFu;
    // PodGroups are homogeneous: most tasks carry exactly the fields of their predecessor.  Comparing the flattened columns of
    // t and t-1 (bit patterns, like the memcmp of the records below) is far cheaper than building and hashing a record.
    auto bits = [](const double* a, size_t i) { uint64_t u; memcpy(&u, a + i, 8); return u; };
    auto same_as_prev = [&](uint32_t t) {
      if (pa && aff_id[t] != aff_id[t - 1]) return false;
      if (aff_as_atoms && (pa_full->task_forbid[t] != pa_full->task_forbid[t - 1] || pa_full->task_contrib[t] != pa_full->task_contrib[t - 1] ||
                           !xg_same(t, t - 1))) return false;
      if (s->task_flags[t] != s->task_flags[t - 1] || s->task_n_aff_terms[t] != s->task_n_aff_terms[t - 1] ||
          s->task_nz_cpu[t] != s->task_nz_cpu[t - 1] || s->task_nz_mem[t] != s->task_nz_mem[t - 1]) return false;
      if (s->task_flags[t] & KB_TASK_HAS_PREFERRED_NODE_AFFINITY) {
        if (!same_pref(pref_of(t), pref_of(t - 1))) return false;
      }
      for (uint32_t r = 0; r < R; ++r) {
        const size_t i = (size_t)r * T + t;
        if (bits(s->task_initreq, i) != bits(s->task_initreq, i - 1) || bits(s->task_resreq, i) != bits(s->task_resreq, i - 1)) return false;
      }
      const uint32_t na = s->task_n_aff_terms[t];
      for (uint32_t w = 0; w < W; ++w) {
        const size_t i = (size_t)w * T + t;
        if (s->task_sel_req[i] != s->task_sel_req[i - 1] || s->task_tol[i] != s->task_tol[i - 1] ||
            s->task_port_own[i] != s->task_port_own[i - 1] || s->task_port_conflict[i] != s->task_port_conflict[i - 1]) return false;
        for (uint32_t a = 0; a < na && a < KB_MAX_AFF_TERMS; ++a) {
          const size_t k = ((size_t)a * W + w) * T + t;
          if (s->task_aff_terms[k] != s->task_aff_terms[k - 1]) return false;
        }
      }
      return true;
    };
    ClassRecBuild rec;                    // the record of the task at hand, reused: clearing 1.3 KB per task would cost more than the rest
    memset(&rec, 0, sizeof rec);
    for (uint32_t t = 0; t < T; ++t) {
      if (t > 0 && prev_class != 0xFFFFFFFFu && same_as_prev(t)) {     // t-1 passed every check below with the same values
        task_class[t] = prev_class; task_empty[t] = task_empty[t - 1];
        continue;
      }
      if ((s->task_flags[t] & KB_TASK_HAS_POD_AFFINITY) && !pa_full)
        return bfail(e, KB_E_UNSUPPORTED_FEATURE, "task %u carries inter-pod affinity terms but the snapshot has no kb_pod_affinity (no CPU fallback)", t);
      if ((s->task_flags[t] & KB_TASK_HAS_PREFERRED_NODE_AFFINITY) && !pa && !will_pipe && !pref_legacy)
        return bfail(e, KB_E_UNSUPPORTED_FEATURE, "task %u carries preferred node-affinity terms: neither the persistent pipeline nor the counter path is available", t);
      ClassPrefBuild cp = pref_of(t);
      if (cp.n) {
        if (cp.n > KB_MAX_PREF_TERMS) return bfail(e, KB_E_BADARG, "task %u: preferred node-affinity arrays missing or n_pref_terms > KB_MAX_PREF_TERMS", t);
        B.has_pref = true;
      }
      if (s->task_n_aff_terms[t] > KB_MAX_AFF_TERMS) return bfail(e, KB_E_BADARG, "task %u: n_aff_terms > KB_MAX_AFF_TERMS", t);
      ClassRecBuild& c = rec;             // every field a task sets is set below; words >= W and dims >= R stay 0
      for (uint32_t r = 0; r < R; ++r) {
        const double ir = s->task_initreq[(size_t)r * T + t], rr = s->task_resreq[(size_t)r * T + t];
        if (r < KB_CLASS_R) { c.initreq[r] = ir; c.resreq[r] = rr; }
        else { hi[r - KB_CLASS_R] = ir; hi[RH + r - KB_CLASS_R] = rr; }
        if (rr > ir) return bfail(e, KB_E_BADARG, "task %u: resreq > initreq in dim %u (violates api/pod_info.go:53-73)", t, r);
      }
      c.nz_cpu = s->task_nz_cpu[t]; c.nz_mem = s->task_nz_mem[t];
      c.n_aff = s->task_n_aff_terms[t];
      c.flags = (s->task_flags[t] & KB_TASK_BEST_EFFORT_QOS) | (pa ? (aff_id[t] << 8) : 0u);      // bits 8.. = aff id: part of the class identity
      for (uint32_t w = 0; w < W; ++w) {
        c.sel_req[w] = s->task_sel_req[(size_t)w * T + t];
        c.tol[w] = s->task_tol[(size_t)w * T + t];
        c.port_own[w] = s->task_port_own[(size_t)w * T + t];
        c.port_conflict[w] = s->task_port_conflict[(size_t)w * T + t];
        c.aff_own[w] = 0;
        for (uint32_t a = 0; a < KB_MAX_AFF_TERMS; ++a) c.aff[a][w] = a < c.n_aff ? s->task_aff_terms[((size_t)a * W + w) * T + t] : 0ull;
      }
      if (aff_as_atoms) {                 // host-level anti-affinity as atoms: forbidden groups conflict, joined groups are set by Allocate
        if (hc.cf.predicates) atoms_of(pa_full->task_forbid[t], t, KB_XGROUP_FORBID, c.port_conflict);
        atoms_of(pa_full->task_contrib[t], t, KB_XGROUP_CONTRIB, c.aff_own);
      }
      task_empty[t] = res_is_empty(R, [&](uint32_t k) { return k < KB_CLASS_R ? c.resreq[k] : hi[RH + k - KB_CLASS_R]; }) ? 1 : 0;   // allocate.go:113-118
      if (prev_class != 0xFFFFFFFFu && same_rec(classes[prev_class], c) && same_pref(class_pref[prev_class], cp) &&
          same_hi(prev_class)) {
        task_class[t] = prev_class; continue; }
      uint64_t h = hash_rec(c);
      if (cp.n) pref_words(cp, [&](uint64_t x) { h = (h ^ x) * 0xFF51AFD7ED558CCDull + (h >> 29); });
      for (uint32_t i = 0; i < 2 * RH; ++i) { uint64_t u; memcpy(&u, &hi[i], 8); h = (h ^ u) * 0xFF51AFD7ED558CCDull + (h >> 29); }
      size_t mask = table.size() - 1, slot = (size_t)h & mask;
      uint32_t found = 0xFFFFFFFFu;
      while (table[slot] != 0xFFFFFFFFu) {
        const uint32_t id = table[slot];
        if (class_hash[id] == h && same_rec(classes[id], c) && same_pref(class_pref[id], cp) && same_hi(id)) { found = id; break; }
        slot = (slot + 1) & mask;
      }
      if (found == 0xFFFFFFFFu) {
        found = (uint32_t)classes.size();
        classes.push_back(c); class_pref.push_back(cp); class_hash.push_back(h);
        class_hi.insert(class_hi.end(), hi.begin(), hi.end());
        table[slot] = found;
        if (classes.size() * 2 > table.size()) {            // grow + rehash
          std::vector<uint32_t> nt(table.size() * 4, 0xFFFFFFFFu);
          const size_t nm = nt.size() - 1;
          for (uint32_t id = 0; id < classes.size(); ++id) { size_t sl = (size_t)class_hash[id] & nm; while (nt[sl] != 0xFFFFFFFFu) sl = (sl + 1) & nm; nt[sl] = id; }
          table.swap(nt);
        }
      }
      task_class[t] = found;
      prev_class = found;
    }
  }
  if (classes.empty()) {
    ClassRecBuild c; memset(&c, 0, sizeof c); classes.push_back(c); ClassPrefBuild cp; memset(&cp, 0, sizeof cp); class_pref.push_back(cp);
    class_hi.assign(2 * (size_t)RH, 0.0);
  }
  // the host copy tests/emu reads, in ClassRec's word capacity (a session with more words runs on the device only)
  if (W <= KB_CLASS_W) {
    B.class_pref.resize(class_pref.size());
    for (size_t k = 0; k < class_pref.size(); ++k) pref_copy(B.class_pref[k], class_pref[k]);
  }
  if (B.has_pref) hc.cf.score_bias += 10ll * (hc.w_nodeaff < 0 ? -(int64_t)hc.w_nodeaff : 0);
  const uint32_t C = (uint32_t)classes.size();
  B.aff = AffDev{};
  std::vector<uint32_t> aff_keyset_off, aff_group_off;
  if (pa) {
    AffDev& A = B.aff;
    A.on = 1; A.n_keysets = pa->n_keysets; A.n_groups = pa->n_groups; A.n_kinds = pa->n_kinds; A.w_podaff = hc.w_podaff;
    for (const ClassAff& ca : aff_tab) if (ca.w_cnt) A.has_weights = 1;
    if (!hc.cf.nodeorder || hc.w_podaff == 0) A.has_weights = 0;          // the priority is not registered / weighs nothing
    if (A.has_weights) hc.cf.score_bias += 10ll * (hc.w_podaff < 0 ? -(int64_t)hc.w_podaff : 0);
    A.has_pref = (B.has_pref && hc.cf.nodeorder) ? 1u : 0u;
    A.has_x = (!aff_xf.empty() || !aff_xc.empty()) ? 1u : 0u;
    aff_keyset_off.assign(pa->n_keysets + 1, 0);
    for (uint32_t k = 0; k < pa->n_keysets; ++k) {
      if (pa->keyset_domains[k] > N) return bfail(e, KB_E_BADARG, "kb_pod_affinity: key set %u has more domains than nodes", k);
      aff_keyset_off[k + 1] = aff_keyset_off[k] + pa->keyset_domains[k];
    }
    A.dom_total = aff_keyset_off[pa->n_keysets];
    aff_group_off.assign(pa->n_groups + 1, 0);
    for (uint32_t g = 0; g < pa->n_groups; ++g) {
      if (pa->group_keyset[g] >= pa->n_keysets) return bfail(e, KB_E_BADARG, "kb_pod_affinity: group %u names a key set out of range", g);
      aff_group_off[g + 1] = aff_group_off[g] + pa->keyset_domains[pa->group_keyset[g]];
    }
    for (uint32_t k = 0; k < pa->n_keysets; ++k)
      for (uint32_t n = 0; n < N; ++n) {
        const int32_t d = pa->node_domain[(size_t)k * N + n];
        if (d < -1 || d >= (int32_t)pa->keyset_domains[k]) return bfail(e, KB_E_BADARG, "kb_pod_affinity: node %u has domain %d under key set %u", n, d, k);
      }
    if (pa->first_unbound_node < -1 || pa->first_unbound_node >= (int32_t)N) return bfail(e, KB_E_BADARG, "kb_pod_affinity: first_unbound_node out of range");
  }

  // ---------------- per-job TaskOrderFn order (session_plugins.go:318-331, priority.go:40-56) ----------------
  std::vector<uint32_t> ord_task, ord_class, job_ord_off(J + 1, 0);
  ord_task.reserve(T);
  for (uint32_t j = 0; j < J; ++j) {
    job_ord_off[j] = (uint32_t)ord_task.size();
    size_t b = ord_task.size();
    for (uint32_t t = s->job_task_off[j]; t < s->job_task_off[j + 1]; ++t) if (!task_empty[t]) ord_task.push_back(t);
    auto before = [&](uint32_t l, uint32_t r) {
      if (hc.task_order_priority && s->task_prio[l] != s->task_prio[r]) return s->task_prio[l] > s->task_prio[r];
      if (s->task_ctime[l] != s->task_ctime[r]) return s->task_ctime[l] < s->task_ctime[r];
      return s->task_uid_rank[l] < s->task_uid_rank[r];
    };
    if (!std::is_sorted(ord_task.begin() + b, ord_task.end(), before)) std::sort(ord_task.begin() + b, ord_task.end(), before);
  }
  job_ord_off[J] = (uint32_t)ord_task.size();
  const uint32_t To = (uint32_t)ord_task.size();
  ord_class.resize(To);
  for (uint32_t i = 0; i < To; ++i) ord_class[i] = task_class[ord_task[i]];

  // ---------------- backfill order (backfill.go:45-47): per job, Pending tasks with an empty InitResreq, UID order ----------------
  std::vector<uint32_t> bf_task, bf_job_off(J + 1, 0), bf_jobs;
  for (uint32_t j = 0; j < J; ++j) {
    bf_job_off[j] = (uint32_t)bf_task.size();
    const size_t b = bf_task.size();
    for (uint32_t t = s->job_task_off[j]; t < s->job_task_off[j + 1]; ++t) {
      const uint32_t id = task_class[t];
      if (res_is_empty(R, [&](uint32_t k) { return init_of(id, k); })) bf_task.push_back(t);
    }
    std::sort(bf_task.begin() + b, bf_task.end(), [&](uint32_t l, uint32_t r) { return s->task_uid_rank[l] < s->task_uid_rank[r]; });
    if (bf_task.size() > b) bf_jobs.push_back(j);
  }
  bf_job_off[J] = (uint32_t)bf_task.size();
  const uint32_t Tb = (uint32_t)bf_task.size();

  // ---------------- slabs ----------------
  const uint32_t NT = (N + TILE_NODES - 1) / TILE_NODES;
  const uint32_t ncols = tile_ncols(R, W);
  const size_t tile_u64 = (size_t)ncols * TILE_NODES;
  Slab& mut = B.mut; Slab& imm = B.imm;
  mut.reset(); imm.reset();
  DevSession H{};            // host view: pointers into the slabs' host buffers
  OffMut& om = B.om; OffImm& oi = B.oi;
  const uint32_t GMAX = std::max(1u, max_grid);
  // shard = a contiguous block of tiles per rank (nodes are in canonical name order)
  const uint32_t tiles_per_rank = (NT + world - 1) / std::max(1u, world);
  B.rank = rank; B.world = std::max(1u, world);
  B.tile_lo = std::min(NT, rank * tiles_per_rank);
  B.tile_hi = std::min(NT, (rank + 1) * tiles_per_rank);
  B.nodes_per_rank = std::max(1u, tiles_per_rank * (uint32_t)TILE_NODES);
  B.tpi = scan_tpi(R, W);
  const uint32_t n_groups = (B.tile_hi - B.tile_lo + B.tpi - 1) / B.tpi;
  // overlap mode (one GPU) keeps one SM for the replayer CTA
  const uint32_t grid = std::max(1u, std::min(n_groups, GMAX > 1 ? GMAX - 1 : GMAX));   // one SM stays free for the replayer CTA
  // persistent pipeline: scanner CTAs keep their tiles resident in shared memory; built for the common record geometry
  // (R = 3, W = 2: cpu, memory, one scalar; 128 label / taint / port atoms) on one GPU (or replicated on every rank)
  B.pipe = 0; B.pipe_S = 0; B.pipe_tpc = 0;
  if (pipe_mode > 0 && world <= 1 && NT > 0 && R == 3 && W == 2 && GMAX >= 2) {
    const size_t tile_bytes = (size_t)ncols * TILE_NODES * 8;
    const uint32_t max_tpc = (uint32_t)((227 * 1024 - 8 * 1024) / tile_bytes);
    const uint32_t smax = GMAX - 1;
    const uint32_t tpc = (NT + smax - 1) / smax;
    if (tpc <= max_tpc) { B.pipe = 1; B.pipe_tpc = tpc; B.pipe_S = (NT + tpc - 1) / tpc; }
  }
  if (B.has_pref && !B.pipe && !B.aff.on && !pref_legacy)
    return bfail(e, KB_E_STATE, "preferred node-affinity terms: the session ended up on the per-launch kernels without the counter path (R = %u, W = %u, %u nodes)", R, W, N);
  om.pipe_g = mut.alloc(sizeof(PipeG));
  om.modlog = mut.alloc(((size_t)To + 64) * 4);
  om.pcand = mut.alloc((size_t)PIPE_RING * std::max(1u, B.pipe_S) * KTOP * 8);
  om.ppref = mut.alloc((size_t)PIPE_RING * std::max(1u, B.pipe_S) * 8);
  om.tiles = mut.alloc(std::max<size_t>(1, NT) * tile_u64 * 8);
  om.used = mut.alloc((size_t)R * std::max(1u, N) * 8);
  om.job_pos = mut.alloc((size_t)std::max(1u, J) * 4);
  om.job_ready = mut.alloc((size_t)std::max(1u, J) * 4);
  om.job_alloc = mut.alloc((size_t)R * std::max(1u, J) * 8);
  om.job_share = mut.alloc((size_t)std::max(1u, J) * 8);
  om.job_placed = mut.alloc((size_t)std::max(1u, J) * 4);
  om.q_head = mut.alloc((size_t)std::max(1u, Q) * 4);
  om.dyn = mut.alloc((size_t)std::max(1u, J) * 4);
  om.q_dyn = mut.alloc((size_t)std::max(1u, Q) * 4);
  om.q_alloc = mut.alloc((size_t)R * std::max(1u, Q) * 8);
  om.q_share = mut.alloc((size_t)std::max(1u, Q) * 8);
  om.qheap = mut.alloc((size_t)std::max(1u, J) * 4);
  om.dec = mut.alloc((size_t)std::max(1u, T) * sizeof(kb_decision));
  om.cand = mut.alloc((size_t)grid * KTOP * 8 * KB_CHAIN_MAX);
  om.ctl = mut.alloc(sizeof(Ctl));
  om.sendbuf = mut.alloc((size_t)xchg_u64(ncols) * 8);
  om.recvbuf = mut.alloc((size_t)std::max(1u, world) * xchg_u64(ncols) * 8);
  om.bf_job_pos = mut.alloc((size_t)std::max(1u, J) * 4);
  om.bf_ctl = mut.alloc(sizeof(Ctl));
  B.rec = rec_kind(R, W);
  const size_t class_bytes = with_rec(B.rec, [](auto t) { return sizeof(typename decltype(t)::type); });
  const size_t pref_bytes = with_rec(B.rec, [](auto t) { return sizeof(ClassPrefOf<typename decltype(t)::type>); });
  oi.classes = imm.alloc((size_t)C * class_bytes);
  oi.total_hi = imm.alloc((size_t)std::max(1u, RH) * 8);
  oi.ord_task = imm.alloc((size_t)std::max(1u, To) * 4);
  oi.ord_class = imm.alloc((size_t)std::max(1u, To) * 4);
  oi.ord_run = imm.alloc((size_t)std::max(1u, To) * 4);
  oi.ord_peek = imm.alloc((size_t)std::max(1u, To) * 4);
  oi.job_ord_off = imm.alloc((size_t)(J + 1) * 4);
  oi.job_min = imm.alloc((size_t)std::max(1u, J) * 4);
  oi.job_queue = imm.alloc((size_t)std::max(1u, J) * 4);
  oi.job_prio = imm.alloc((size_t)std::max(1u, J) * 4);
  oi.job_tb = imm.alloc((size_t)std::max(1u, J) * 4);
  oi.q_static = imm.alloc((size_t)std::max(1u, J) * 4);
  oi.q_static_off = imm.alloc((size_t)(Q + 1) * 4);
  oi.q_des = imm.alloc((size_t)R * std::max(1u, Q) * 8);
  oi.q_des_p = imm.alloc((size_t)std::max(1u, Q) * 4);
  oi.q_ctime = imm.alloc((size_t)std::max(1u, Q) * 8);
  oi.task_class = imm.alloc((size_t)std::max(1u, T) * 4);
  oi.job_ready0 = imm.alloc((size_t)std::max(1u, J) * 4);
  oi.bf_ord_task = imm.alloc((size_t)std::max(1u, Tb) * 4);
  oi.bf_ord_class = imm.alloc((size_t)std::max(1u, Tb) * 4);
  oi.bf_ord_run = imm.alloc((size_t)std::max(1u, Tb) * 4);
  oi.bf_ord_peek = imm.alloc((size_t)std::max(1u, Tb) * 4);
  oi.bf_job_ord_off = imm.alloc((size_t)(J + 1) * 4);
  oi.bf_jobs = imm.alloc((size_t)std::max<size_t>(1, bf_jobs.size()) * 4);
  oi.bf_jobs_off = imm.alloc(2 * 4);
  oi.bf_classes = imm.alloc((size_t)(Tb ? C : 1) * class_bytes);
  oi.ord_chain = imm.alloc((size_t)std::max(1u, To) * (KB_CHAIN_MAX - 1) * 4);
  oi.class_pref = imm.alloc((size_t)(B.has_pref ? C : 1) * pref_bytes);
  if (pa) {
    oi.aff_node_domain = imm.alloc((size_t)std::max(1u, pa->n_keysets) * std::max(1u, N) * 4);
    oi.aff_keyset_off = imm.alloc((size_t)(pa->n_keysets + 1) * 4);
    oi.aff_group_keyset = imm.alloc((size_t)std::max(1u, pa->n_groups) * 4);
    oi.aff_group_off = imm.alloc((size_t)(pa->n_groups + 1) * 4);
    oi.aff_cls = imm.alloc((size_t)C * sizeof(ClassAff));
    oi.aff_w_kind = imm.alloc(std::max<size_t>(1, aff_wk.size()) * 4);
    oi.aff_w_keyset = imm.alloc(std::max<size_t>(1, aff_wk.size()) * 4);
    oi.aff_w_value = imm.alloc(std::max<size_t>(1, aff_wk.size()) * 8);
    oi.aff_kind_unbound = imm.alloc(std::max(1u, pa->n_kinds));
    oi.aff_xf = imm.alloc(std::max<size_t>(1, aff_xf.size()) * sizeof(AffX));
    oi.aff_xc = imm.alloc(std::max<size_t>(1, aff_xc.size()) * 4);
    om.aff_cnt = mut.alloc((size_t)std::max(1u, aff_group_off[pa->n_groups]) * 4);
    om.aff_total = mut.alloc((size_t)std::max(1u, pa->n_groups) * 4);
    om.aff_kind_count = mut.alloc((size_t)std::max(1u, pa->n_kinds) * std::max(1u, N) * 4);
    om.aff_first_unbound = mut.alloc(8);
    om.aff_dom_sum = mut.alloc((size_t)std::max(1u, B.aff.dom_total) * 8);
    om.aff_minmax = mut.alloc(32);
  }
  mut.commit(); imm.commit();

  B.R = R; B.W = W; B.N = N; B.T = T; B.J = J; B.Q = Q; B.C = C; B.NT = NT; B.ncols = ncols; B.To = To; B.Tb = Tb;
  B.bind(H, mut.host.data(), imm.host.data());

  // ---------------- node tiles ----------------
  for (uint32_t t = 0; t < NT; ++t) {
    uint64_t* tb = H.tiles + (size_t)t * tile_u64;
    for (uint32_t i = 0; i < TILE_NODES; ++i) {
      const uint32_t n = t * TILE_NODES + i;
      auto put = [&](uint32_t c, uint64_t v) { tb[(size_t)c * TILE_NODES + i] = v; };
      if (n < N) {
        for (uint32_t r = 0; r < R; ++r) {
          put(col_idle(R, r), double_as_u64(s->node_idle[(size_t)r * N + n]));
          put(col_rel(R, r), double_as_u64(s->node_releasing[(size_t)r * N + n]));
          H.node_used[(size_t)r * N + n] = s->node_used[(size_t)r * N + n];
        }
        put(col_alloc_cpu(R), (uint64_t)s->node_alloc_cpu[n]); put(col_alloc_mem(R), (uint64_t)s->node_alloc_mem[n]);
        put(col_nz_cpu(R), (uint64_t)s->node_nz_cpu[n]); put(col_nz_mem(R), (uint64_t)s->node_nz_mem[n]);
        put(col_pods(R), (uint64_t)(uint32_t)s->node_pods[n] | ((uint64_t)(uint32_t)s->node_max_pods[n] << 32));
        // KB_SNAPSHOT_LISTED_POD_WITHOUT_NODE: InterPodAffinityMatches errors for every pair, i.e. the predicates plugin rejects
        // every node; K1 reads that as a node condition that fails (only evaluated when the plugin's predicate is enabled)
        uint64_t no_scalars = (s->node_alloc_present[n] & ~3u) == 0 ? (NODE_IDLE_NO_SCALARS | NODE_REL_NO_SCALARS) : 0ull;
        for (uint32_t r = 2; r < R; ++r) {
          if (s->node_idle[(size_t)r * N + n] != 0) no_scalars &= ~NODE_IDLE_NO_SCALARS;
          if (s->node_releasing[(size_t)r * N + n] != 0) no_scalars &= ~NODE_REL_NO_SCALARS;
        }
        put(col_flags(R), (uint64_t)s->node_flags[n] | ((s->flags & KB_SNAPSHOT_LISTED_POD_WITHOUT_NODE) ? (uint64_t)KB_NODE_NOT_READY : 0ull) |
                          no_scalars);
        for (uint32_t w = 0; w < W; ++w) {
          put(col_labels(R, W, w), s->node_labels[(size_t)w * N + n]);
          put(col_taints(R, W, w), s->node_taints[(size_t)w * N + n]);
          put(col_ports(R, W, w), s->node_ports[(size_t)w * N + n] | (aff_as_atoms ? node_aff_bits[(size_t)w * N + n] : 0ull));
        }
      } else {                                   // padding node: can never fit (kernels also test node < N)
        for (uint32_t r = 0; r < R; ++r) { put(col_idle(R, r), double_as_u64(-1e300)); put(col_rel(R, r), double_as_u64(-1e300)); }
        put(col_flags(R), (uint64_t)KB_NODE_UNSCHEDULABLE);
      }
    }
  }

  // ---------------- immutable job / queue / class tables ----------------
  // the class table in the session's record type; a wide record joins the narrow part with its dims past KB_CLASS_R
  auto write_classes = [&](unsigned char* dst, const bool backfill) {
    with_rec(B.rec, [&](auto t) {
      using CR = typename decltype(t)::type;
      for (uint32_t k = 0; k < C; ++k) {
        CR w;
        memset(&w, 0, sizeof w);
        class_copy(w, classes[k]);
        for (uint32_t r = KB_CLASS_R; r < R && r < CR::CAP; ++r) {
          w.initreq[r] = class_hi[(size_t)k * 2 * RH + (r - KB_CLASS_R)];
          w.resreq[r] = class_hi[(size_t)k * 2 * RH + RH + (r - KB_CLASS_R)];
        }
        if (backfill) for (uint32_t r = 0; r < CR::CAP; ++r) w.initreq[r] = w.resreq[r];
        memcpy(dst + k * sizeof w, &w, sizeof w);
      }
    });
  };
  write_classes(imm.host.data() + oi.classes, false);
  if (B.has_pref)
    with_rec(B.rec, [&](auto t) {
      auto* d = reinterpret_cast<ClassPrefOf<typename decltype(t)::type>*>(imm.host.data() + oi.class_pref);
      for (uint32_t k = 0; k < C; ++k) pref_copy(d[k], class_pref[k]);
    });
  if (pa) {
    unsigned char* ib = imm.host.data(); unsigned char* mb = mut.host.data();
    if (pa->n_keysets && N) memcpy(ib + oi.aff_node_domain, pa->node_domain, (size_t)pa->n_keysets * N * 4);
    memcpy(ib + oi.aff_keyset_off, aff_keyset_off.data(), aff_keyset_off.size() * 4);
    if (pa->n_groups) memcpy(ib + oi.aff_group_keyset, pa->group_keyset, (size_t)pa->n_groups * 4);
    memcpy(ib + oi.aff_group_off, aff_group_off.data(), aff_group_off.size() * 4);
    std::vector<uint8_t> keyset_single(std::max(1u, pa->n_keysets), 1);      // every domain of the key set is ONE node
    for (uint32_t k = 0; k < pa->n_keysets; ++k) {
      std::vector<uint32_t> size(std::max(1u, pa->keyset_domains[k]), 0);
      for (uint32_t n = 0; n < N; ++n) { const int32_t d = pa->node_domain[(size_t)k * N + n]; if (d >= 0 && ++size[d] > 1) keyset_single[k] = 0; }
    }
    ClassAff* hca = (ClassAff*)(ib + oi.aff_cls);
    for (uint32_t k = 0; k < C; ++k) {
      const uint32_t id = classes[k].flags >> 8;
      if (id < aff_tab.size()) hca[k] = aff_tab[id]; else { memset(&hca[k], 0, sizeof(ClassAff)); hca[k].need = -1; hca[k].kind = -1; }
      if (!B.aff.has_weights) { hca[k].w_cnt = 0; hca[k].w_keysets = 0; }
      if (!hc.cf.predicates) { hca[k].forbid = 0; hca[k].xf_cnt = 0; hca[k].xs_cnt = 0; hca[k].need = -1; }   // step 10 belongs to the predicates plugin
      // groups the class both joins and reads: if all of them live on single-node domains (and the needed group is not among
      // them: its `total` would end the first-of-series escape for every node), its own placements only change the chosen node
      const int32_t need = hca[k].need;
      const uint64_t needbit = (need >= 0 && need < 64) ? (1ull << need) : 0ull;
      bool need_joined = (hca[k].contrib & needbit) != 0;
      for (uint32_t i = 0; i < hca[k].xc_cnt && need >= 64; ++i) need_joined = need_joined || aff_xc[hca[k].xc_off + i] == (uint32_t)need;
      uint64_t m = hca[k].contrib & (hca[k].forbid | needbit);
      bool multi = !need_joined;
      while (m && multi) {
        const uint32_t g = (uint32_t)__builtin_ctzll(m);
        m &= m - 1;
        multi = keyset_single[pa->group_keyset[g]] != 0;
      }
      for (uint32_t i = 0; i < hca[k].xs_cnt && multi; ++i) multi = keyset_single[pa->group_keyset[aff_xf_group[hca[k].xf_off + i]]] != 0;
      hca[k].pred_multi_ok = multi ? 1u : 0u;
      hca[k].self_block = (multi && ((hca[k].contrib & hca[k].forbid) != 0 || hca[k].xs_cnt != 0)) ? 1 : 0;
    }
    if (!aff_wk.empty()) {
      memcpy(ib + oi.aff_w_kind, aff_wk.data(), aff_wk.size() * 4); memcpy(ib + oi.aff_w_keyset, aff_wks.data(), aff_wks.size() * 4);
      memcpy(ib + oi.aff_w_value, aff_wv.data(), aff_wv.size() * 8);
    }
    if (pa->n_kinds) memcpy(ib + oi.aff_kind_unbound, pa->kind_unbound, pa->n_kinds);
    if (!aff_xf.empty()) memcpy(ib + oi.aff_xf, aff_xf.data(), aff_xf.size() * sizeof(AffX));
    if (!aff_xc.empty()) memcpy(ib + oi.aff_xc, aff_xc.data(), aff_xc.size() * 4);
    if (aff_group_off[pa->n_groups]) memcpy(mb + om.aff_cnt, pa->group_count0, (size_t)aff_group_off[pa->n_groups] * 4);
    if (pa->n_groups) memcpy(mb + om.aff_total, pa->group_total0, (size_t)pa->n_groups * 4);
    if (pa->n_kinds && N) memcpy(mb + om.aff_kind_count, pa->node_kind_count0, (size_t)pa->n_kinds * N * 4);
    *(int32_t*)(mb + om.aff_first_unbound) = pa->first_unbound_node;
  }
  if (To) { memcpy(H.ord_task, ord_task.data(), (size_t)To * 4); memcpy(H.ord_class, ord_class.data(), (size_t)To * 4); }
  for (uint32_t j = 0; j < J; ++j)                     // run lengths, right to left inside each job
    for (uint32_t i = job_ord_off[j + 1]; i-- > job_ord_off[j];)
      H.ord_run[i] = (i + 1 < job_ord_off[j + 1] && ord_class[i + 1] == ord_class[i]) ? H.ord_run[i + 1] + 1 : 1;
  memcpy(H.job_ord_off, job_ord_off.data(), (size_t)(J + 1) * 4);
  if (T) memcpy(imm.host.data() + oi.task_class, task_class.data(), (size_t)T * 4);
  std::vector<uint32_t> tb_order(J);
  for (uint32_t j = 0; j < J; ++j) tb_order[j] = j;
  {
    auto before = [&](uint32_t l, uint32_t r) {
      if (s->job_ctime[l] != s->job_ctime[r]) return s->job_ctime[l] < s->job_ctime[r];
      return l < r;
    };
    if (!std::is_sorted(tb_order.begin(), tb_order.end(), before)) std::sort(tb_order.begin(), tb_order.end(), before);
  }
  for (uint32_t i = 0; i < J; ++i) H.job_tb_rank[tb_order[i]] = i;
  int32_t* h_ready0 = (int32_t*)(imm.host.data() + oi.job_ready0);
  for (uint32_t j = 0; j < J; ++j) {
    H.job_min_avail[j] = s->job_min_avail[j];
    H.job_queue[j] = s->job_queue[j];
    H.job_prio[j] = s->job_prio[j];
    H.job_ready[j] = s->job_ready0[j];
    h_ready0[j] = s->job_ready0[j];
    H.job_pos[j] = job_ord_off[j];
    for (uint32_t r = 0; r < R; ++r) H.job_alloc[(size_t)r * J + j] = s->job_alloc0[(size_t)r * J + j];
  }
  for (uint32_t q = 0; q < Q; ++q) H.q_ctime[q] = s->queue_ctime[q];

  // drf OnSessionOpen (drf.go:60-83): total = sum of node Allocatable; share per job
  H.total_dims_mask = 3u;
  for (uint32_t r = 0; r < KB_MAX_R; ++r) B.total[r] = 0;
  for (uint32_t n = 0; n < N; ++n) {
    H.total_dims_mask |= s->node_alloc_present[n] & ~3u;
    for (uint32_t r = 0; r < R; ++r)
      if (r < 2 || ((s->node_alloc_present[n] >> r) & 1u)) B.total[r] += s->node_allocatable[(size_t)r * N + n];
  }
  H.total_dims_mask &= (R >= 32 ? 0xFFFFFFFFu : ((1u << R) - 1u));
  B.total_dims_mask = H.total_dims_mask;
  for (uint32_t r = 0; r < R && r < KB_CLASS_R; ++r) H.total[r] = B.total[r];
  if (KB_CLASS_R < KB_MAX_R)
    for (uint32_t i = 0; i < RH; ++i) reinterpret_cast<double*>(imm.host.data() + oi.total_hi)[i] = B.total[KB_CLASS_R + i];
  for (uint32_t j = 0; j < J; ++j) {
    if (!hc.drf_present) H.job_share[j] = 0.0;
    else with_rec(B.rec, [&](auto t) { update_job_share<decltype(t)::type::CAP>(H, j); });
  }

  // proportion OnSessionOpen (proportion.go:58-154)
  B.q_alloc_present.assign(std::max(1u, Q), 0);
  if (hc.proportion_present) {
    struct Attr { bool used = false; int32_t weight = 0; HostRes deserved, allocated, request; };
    std::vector<Attr> qa(Q);
    HostRes total; total.present = H.total_dims_mask & ~3u;
    for (uint32_t r = 0; r < R; ++r) total.v[r] = B.total[r];
    for (uint32_t j = 0; j < J; ++j) {                                   // :67-98
      Attr& a = qa[s->job_queue[j]];
      if (!a.used) { a.used = true; a.weight = s->queue_weight[s->job_queue[j]]; }
      HostRes al; al.present = s->job_alloc0_present[j] & ~3u;
      for (uint32_t r = 0; r < R; ++r) al.v[r] = (r < 2 || ((al.present >> r) & 1u)) ? s->job_alloc0[(size_t)r * J + j] : 0.0;
      hr_add(R, a.allocated, al); hr_add(R, a.request, al);
      for (uint32_t t = s->job_task_off[j]; t < s->job_task_off[j + 1]; ++t) {
        HostRes rq; rq.present = s->task_res_present[t] & ~3u;
        for (uint32_t r = 0; r < R; ++r) rq.v[r] = (r < 2 || ((rq.present >> r) & 1u)) ? s->task_resreq[(size_t)r * T + t] : 0.0;
        hr_add(R, a.request, rq);
      }
    }
    HostRes remaining = total;                                           // :100
    std::vector<uint32_t> active;                                        // used queues that have not met their request, ascending
    for (uint32_t q = 0; q < Q; ++q) if (qa[q].used) active.push_back(q);
    for (;;) {
      int32_t totalWeight = 0;
      for (const uint32_t q : active) totalWeight += qa[q].weight;
      if (totalWeight == 0) break;
      HostRes incD, decD;
      size_t keep = 0;
      for (const uint32_t q : active) {
        Attr& a = qa[q];
        HostRes old = a.deserved;
        HostRes part = remaining;
        const double ratio = (double)a.weight / (double)totalWeight;
        part.v[0] = part.v[0] * ratio; part.v[1] = part.v[1] * ratio;
        for (uint32_t k = 2; k < R; ++k) if ((part.present >> k) & 1u) part.v[k] = part.v[k] * ratio;
        hr_add(R, a.deserved, part);
        if (hr_less(R, a.request, a.deserved)) a.deserved = hr_min(R, a.deserved, a.request);
        else active[keep++] = q;
        HostRes inc, dec;
        hr_diff(R, a.deserved, old, inc, dec);
        hr_add(R, incD, inc); hr_add(R, decD, dec);
      }
      active.resize(keep);
      if (!hr_sub(R, remaining, incD)) return bfail(e, KB_E_STATE, "proportion: remaining.Sub would panic in the reference (resource_info.go:158)");
      hr_add(R, remaining, decD);
      if (hr_is_empty(R, remaining)) break;
    }
    for (uint32_t q = 0; q < Q; ++q) {
      H.q_deserved_present[q] = qa[q].deserved.present;
      B.q_alloc_present[q] = qa[q].allocated.present;
      for (uint32_t r = 0; r < R; ++r) {
        H.q_deserved[(size_t)r * Q + q] = (r < 2 || ((qa[q].deserved.present >> r) & 1u)) ? qa[q].deserved.v[r] : 0.0;
        H.q_allocated[(size_t)r * Q + q] = (r < 2 || ((qa[q].allocated.present >> r) & 1u)) ? qa[q].allocated.v[r] : 0.0;
      }
      update_queue_share(H, q);
    }
  }

  // ---------------- job lists per queue, queue heap, first visit (allocate.go:47-65, 89-126) ----------------
  {
    std::vector<uint32_t> cnt(Q + 1, 0);
    for (uint32_t j = 0; j < J; ++j) cnt[s->job_queue[j] + 1]++;
    for (uint32_t q = 0; q < Q; ++q) cnt[q + 1] += cnt[q];
    memcpy(H.q_static_off, cnt.data(), (size_t)(Q + 1) * 4);
    std::vector<uint32_t> fill(cnt.begin(), cnt.end() - 1);
    std::vector<uint32_t> next_diff(std::max(1u, To), 0xFFFFFFFFu);     // first later slot (static walk) with another class
    const bool want_chain = world <= 1 && (kchain == 2 || kchain == 4 || B.pipe);
    const bool want_peek = world <= 1 && (overlap_mode > 0 || (overlap_mode < 0 && N >= 65536 && Q == 1));
    for (uint32_t j = 0; j < J; ++j) H.q_static[fill[s->job_queue[j]]++] = j;
    for (uint32_t q = 0; q < Q; ++q) {
      {
        auto before = [&](uint32_t l, uint32_t r) { return job_before(H, l, r); };
        if (!std::is_sorted(H.q_static + cnt[q], H.q_static + cnt[q + 1], before)) std::sort(H.q_static + cnt[q], H.q_static + cnt[q + 1], before);
      }
      H.q_static_head[q] = cnt[q];
      if (!want_peek && !want_chain) continue;      // the prediction tables are only read by the overlap / chained-visit kernels
      // prediction table: walking the queue's static job order backwards, the first class that differs from a slot's own
      uint32_t next_slot = 0xFFFFFFFFu;
      for (uint32_t k = cnt[q + 1]; k-- > cnt[q];) {
        const uint32_t j = H.q_static[k];
        for (uint32_t i = job_ord_off[j + 1]; i-- > job_ord_off[j];) {
          if (next_slot == 0xFFFFFFFFu) { H.ord_peek[i] = 0xFFFFFFFFu; next_diff[i] = 0xFFFFFFFFu; }
          else {
            H.ord_peek[i] = (ord_class[next_slot] != ord_class[i]) ? ord_class[next_slot] : H.ord_peek[next_slot];
            next_diff[i] = (ord_class[next_slot] != ord_class[i]) ? next_slot : next_diff[next_slot];
          }
          // chain: classes of the following runs, each different from every class before it in the chain
          uint32_t seen[KB_CHAIN_MAX] = {ord_class[i]};
          uint32_t ns = 1, sl = next_diff[i];
          for (uint32_t c = 0; c + 1 < KB_CHAIN_MAX; ++c) {
            uint32_t cls = 0xFFFFFFFFu;
            if (sl != 0xFFFFFFFFu && ns == c + 1) {
              cls = ord_class[sl];
              for (uint32_t z = 0; z < ns; ++z) if (seen[z] == cls) cls = 0xFFFFFFFFu;     // a repeat ends the chain
              if (cls != 0xFFFFFFFFu) { seen[ns++] = cls; sl = next_diff[sl]; }
            }
            H.ord_chain[(size_t)i * (KB_CHAIN_MAX - 1) + c] = cls;
          }
          next_slot = i;
        }
      }
    }
  }
  // overlap pays when the scan side (several tile groups per CTA + a wide merge) rivals the replay side
  B.overlap = (world <= 1) ? (overlap_mode < 0 ? ((N >= 65536 && Q == 1) ? 1u : 0u) : (uint32_t)overlap_mode) : 0u;
  if (B.has_pref) B.overlap = 0;
  B.kchain = (world <= 1 && !B.overlap && (kchain == 2 || kchain == 4)) ? kchain : 1u;
  H.kchain = B.kchain;
  Ctl& c0 = *H.ctl;
  memset(&c0, 0, sizeof c0);
  c0.cur_job = -1;
  for (uint32_t j = 0; j < J; ++j) qheap_push(H, c0, s->job_queue[j]);      // one push PER JOB (allocate.go:52)
  for (uint32_t t = 0; t < T; ++t) {
    kb_decision d; d.node = -1; d.kind = task_empty[t] ? KB_KIND_SKIPPED : KB_KIND_NONE; d.dispatched = 0; d.reserved = 0;
    d.step = 0xFFFFFFFFu; d.dispatch_step = 0xFFFFFFFFu;
    H.dec[t] = d;
  }
  select_next_visit(H, c0);
  c0.scan_class = c0.cur_class;      // the first launch has no list yet: scan for the first visit, nothing excluded
  c0.n_excl = 0; c0.list_valid = 0; c0.patch_valid = 0;
  c0.xchg_epoch = 1;
  publish_chain(H, c0);

  // ---------------- backfill view: order tables, cursors, first visit ----------------
  {
    DevSession HB{};
    B.bind_backfill(HB, mut.host.data(), imm.host.data());
    if (Tb) write_classes(imm.host.data() + oi.bf_classes, true);
    for (uint32_t i = 0; i < Tb; ++i) { HB.ord_task[i] = bf_task[i]; HB.ord_class[i] = task_class[bf_task[i]]; HB.ord_peek[i] = 0xFFFFFFFFu; }
    for (uint32_t j = 0; j < J; ++j) {
      for (uint32_t i = bf_job_off[j + 1]; i-- > bf_job_off[j];)
        HB.ord_run[i] = (i + 1 < bf_job_off[j + 1] && HB.ord_class[i + 1] == HB.ord_class[i]) ? HB.ord_run[i + 1] + 1 : 1;
      HB.job_pos[j] = bf_job_off[j];
    }
    memcpy(HB.job_ord_off, bf_job_off.data(), (size_t)(J + 1) * 4);
    for (size_t i = 0; i < bf_jobs.size(); ++i) HB.q_static[i] = bf_jobs[i];
    HB.q_static_off[0] = 0; HB.q_static_off[1] = (uint32_t)bf_jobs.size();
    Ctl& cb = *HB.ctl;
    memset(&cb, 0, sizeof cb);
    cb.cur_job = -1;
    select_next_visit(HB, cb);
    cb.scan_class = cb.cur_class;
    cb.xchg_epoch = 1;
  }

  B.R = R; B.W = W; B.N = N; B.T = T; B.J = J; B.Q = Q; B.C = C; B.NT = NT; B.ncols = ncols; B.To = To; B.grid = grid;
  B.job_min_avail.assign(s->job_min_avail, s->job_min_avail + J);
  return KB_OK;
}

}  // namespace kb
#endif  // KB_BUILD_H_
