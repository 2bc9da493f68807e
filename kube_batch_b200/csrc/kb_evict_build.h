// kb_evict_build.h — CUDA-free host-side construction of the evict path's data (kb_evict.h) from kb_running + the built
// session: Running tasks CSR by node (UID order inside a node), every job's Pending tasks in TaskOrderFn order, the job heaps
// of the queues and reclaim's queue heap (filled by evict_init at the start of each action, like reclaim.go:53-81 / preempt.go:54-75).
// Used by kb_engine.cu (uploads the two slabs) and by tests/emu (runs them on the CPU).
#ifndef KB_EVICT_BUILD_H_
#define KB_EVICT_BUILD_H_

#include "kb_build.h"
#include "kb_evict.h"

namespace kb {

struct EvictBuilt {
  Slab imm, mut;
  struct { size_t node_off, r_orig, r_job, r_resreq, r_present, r_prio, r_ctime, r_uid_rank, r_flags, pt_task, pt_off, task_class, task_present, job_waiting0,
                 r_atom_off, r_atom, atom_bit, atom_local; } oi;
  struct { size_t r_state, pt_pos, job_waiting, jheap, jheap_len, qheap, queue_map, q_alloc_present, evict_order, ops, scratch, ctl, atom_cnt; } om;
  uint32_t n_run = 0, Tall = 0;
  bool lists = false;                // kb_running carried aff_group_off: the atoms of the members are counted
  bool groups_unread = false;        // BuiltSession.aff_groups_unread: a member's eviction changes nothing observable (empty atom lists)
  uint32_t n_atoms = 0;
  EvictConf ec{};
  void bind(EvictDev& E, unsigned char* ib, unsigned char* mb) const {
    E.ec = ec; E.n_run = n_run; E.Tall = Tall;
    E.node_off = (const uint32_t*)(ib + oi.node_off); E.r_orig = (const uint32_t*)(ib + oi.r_orig); E.r_job = (const uint32_t*)(ib + oi.r_job);
    E.r_resreq = (const double*)(ib + oi.r_resreq); E.r_present = (const uint32_t*)(ib + oi.r_present); E.r_prio = (const int32_t*)(ib + oi.r_prio);
    E.r_ctime = (const int64_t*)(ib + oi.r_ctime); E.r_uid_rank = (const uint32_t*)(ib + oi.r_uid_rank); E.r_flags = (const uint32_t*)(ib + oi.r_flags);
    E.pt_task = (const uint32_t*)(ib + oi.pt_task); E.pt_off = (const uint32_t*)(ib + oi.pt_off);
    E.task_class = (const uint32_t*)(ib + oi.task_class); E.task_present = (const uint32_t*)(ib + oi.task_present);
    E.job_waiting0 = (const int32_t*)(ib + oi.job_waiting0);
    E.n_atoms = n_atoms;
    E.r_atom_off = (lists || groups_unread) ? (const uint32_t*)(ib + oi.r_atom_off) : nullptr; E.r_atom = (const uint32_t*)(ib + oi.r_atom);
    E.atom_bit = (const uint32_t*)(ib + oi.atom_bit); E.atom_local = (const int32_t*)(ib + oi.atom_local);
    E.atom_cnt = (int32_t*)(mb + om.atom_cnt);
    E.r_state = (uint8_t*)(mb + om.r_state); E.pt_pos = (uint32_t*)(mb + om.pt_pos); E.job_waiting = (int32_t*)(mb + om.job_waiting);
    E.jheap = (uint32_t*)(mb + om.jheap); E.jheap_len = (uint32_t*)(mb + om.jheap_len); E.qheap = (uint32_t*)(mb + om.qheap);
    E.queue_map = (uint32_t*)(mb + om.queue_map);
    E.q_alloc_present = (uint32_t*)(mb + om.q_alloc_present); E.evict_order = (uint32_t*)(mb + om.evict_order);
    E.ops = (uint32_t*)(mb + om.ops); E.scratch = (uint32_t*)(mb + om.scratch); E.ctl = (EvictCtl*)(mb + om.ctl);
  }
};

// H: the session's DevSession bound to the HOST slabs of `B` in their as-loaded state (the comparators read it).
inline int build_evict(const kb_snapshot* s, const kb_running* run, const BuiltSession& B, const DevSession& H, EvictBuilt& EB, BuildErr* e) {
  const uint32_t R = s->R, N = s->N, T = s->T, J = s->J, Q = s->Q;
  const uint32_t n = run ? run->n : 0;
  if (n && (!run->node || !run->job || !run->resreq || !run->res_present || !run->prio || !run->ctime || !run->uid_rank || !run->flags))
    return bfail(e, KB_E_BADARG, "kb_running: NULL array");
  for (uint32_t i = 0; i < n; ++i) {
    if (run->node[i] >= N || run->job[i] >= J) return bfail(e, KB_E_BADARG, "kb_running[%u]: node / job index out of range", i);
    if (s->job_ready0[run->job[i]] <= 0) return bfail(e, KB_E_BADARG, "kb_running[%u]: job_ready0 of job %u does not cover its running tasks", i, run->job[i]);
  }
  // ---- the counter groups of every Running member (kb_running.aff_group_off / aff_group) ----
  const kb_pod_affinity* pa = s->pod_affinity;
  const uint32_t NG = pa ? pa->n_groups : 0u;
  const bool lists = run && run->aff_group_off;
  const uint32_t* go = lists ? run->aff_group_off : nullptr;
  if (lists) {
    for (uint32_t i = 0; i < n; ++i)
      if (go[i] > go[i + 1]) return bfail(e, KB_E_BADARG, "kb_running: aff_group_off is not monotone at task %u", i);
    if (go[n] > go[0] && !run->aff_group) return bfail(e, KB_E_BADARG, "kb_running: aff_group is NULL but aff_group_off names entries");
    // per (group, domain): listed Running members <= group_count0 (it counts every AllocatedStatus member)
    std::vector<uint32_t> gbase(NG + 1, 0);
    for (uint32_t g = 0; g < NG; ++g) gbase[g + 1] = gbase[g] + pa->keyset_domains[pa->group_keyset[g]];
    std::vector<uint64_t> keys;
    for (uint32_t i = 0; i < n; ++i)
      for (uint32_t k = go[i]; k < go[i + 1]; ++k) {
        const uint32_t g = run->aff_group[k];
        if (g >= NG) return bfail(e, KB_E_BADARG, "kb_running[%u]: aff_group entry %u names group %u, the session has %u", i, k, g, NG);
        const int32_t d = pa->node_domain[(size_t)pa->group_keyset[g] * N + run->node[i]];
        if (d >= 0) keys.push_back((uint64_t)gbase[g] + (uint32_t)d);
      }
    std::sort(keys.begin(), keys.end());
    for (size_t a = 0, b; a < keys.size(); a = b) {
      for (b = a; b < keys.size() && keys[b] == keys[a]; ++b) {}
      if ((int64_t)(b - a) > (int64_t)pa->group_count0[keys[a]])
        return bfail(e, KB_E_BADARG, "kb_running: %zu Running members listed in one domain of a counter group whose group_count0 there is %d", b - a, pa->group_count0[keys[a]]);
    }
  }
  EB.n_run = n;
  EB.lists = lists;
  EB.groups_unread = B.aff_groups_unread;      // r_atom_off stays all zero without lists: no member has an atom
  EB.ec.reclaim_fns = B.hc.reclaim_fns; EB.ec.preempt_fns = B.hc.preempt_fns;
  EB.ec.gang_pipelined = B.hc.gang_pipelined ? 1u : 0u; EB.ec.task_order_priority = B.hc.task_order_priority ? 1u : 0u;
  // ---- Running tasks: CSR by node, UID order inside a node ----
  std::vector<uint32_t> order(n);
  for (uint32_t i = 0; i < n; ++i) order[i] = i;
  std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) {
    if (run->node[a] != run->node[b]) return run->node[a] < run->node[b];
    return run->uid_rank[a] < run->uid_rank[b];
  });
  // ---- every job's Pending tasks in TaskOrderFn order (session_plugins.go:318-331; priority.go:40-56) ----
  std::vector<uint32_t> pt(T), pt_off(J + 1, 0);
  for (uint32_t j = 0; j < J; ++j) {
    const uint32_t b = s->job_task_off[j], en = s->job_task_off[j + 1];
    pt_off[j] = b;
    for (uint32_t t = b; t < en; ++t) pt[t] = t;
    auto before = [&](uint32_t l, uint32_t r) {
      if (B.hc.task_order_priority && s->task_prio[l] != s->task_prio[r]) return s->task_prio[l] > s->task_prio[r];
      if (s->task_ctime[l] != s->task_ctime[r]) return s->task_ctime[l] < s->task_ctime[r];
      return s->task_uid_rank[l] < s->task_uid_rank[r];
    };
    std::sort(pt.begin() + b, pt.begin() + en, before);
  }
  pt_off[J] = T;
  EB.Tall = T;

  // local atom index of each port-word bit some member's group became (kb_build.h); groups that are no atom are dropped: nobody
  // reads or joins them, so their members' evictions change nothing observable
  std::vector<int32_t> atom_local((size_t)64 * B.W, -1);          // one entry per port-word bit of the session
  std::vector<uint32_t> atom_bit, r_atom_off(1, 0), r_atom;
  if (lists) {
    std::vector<uint32_t> mine;
    for (uint32_t k = 0; k < n; ++k) {
      const uint32_t i = order[k];
      mine.clear();
      for (uint32_t x = go[i]; x < go[i + 1]; ++x) {
        const uint32_t g = run->aff_group[x];
        const int32_t a = g < B.aff_atom_of_group.size() ? B.aff_atom_of_group[g] : -1;
        if (a < 0) continue;
        if (atom_local[a] < 0) { atom_local[a] = (int32_t)atom_bit.size(); atom_bit.push_back((uint32_t)a); }
        mine.push_back((uint32_t)atom_local[a]);
      }
      std::sort(mine.begin(), mine.end());
      mine.erase(std::unique(mine.begin(), mine.end()), mine.end());
      r_atom.insert(r_atom.end(), mine.begin(), mine.end());
      r_atom_off.push_back((uint32_t)r_atom.size());
    }
  }
  const uint32_t NA = (uint32_t)atom_bit.size();
  EB.n_atoms = NA;

  Slab& imm = EB.imm; Slab& mut = EB.mut;
  imm.reset(); mut.reset();
  const size_t n1 = std::max(1u, n), T1 = std::max(1u, T), J1 = std::max(1u, J), Q1 = std::max(1u, Q);
  EB.oi.node_off = imm.alloc(((size_t)N + 1) * 4); EB.oi.r_orig = imm.alloc(n1 * 4); EB.oi.r_job = imm.alloc(n1 * 4);
  EB.oi.r_resreq = imm.alloc((size_t)R * n1 * 8); EB.oi.r_present = imm.alloc(n1 * 4); EB.oi.r_prio = imm.alloc(n1 * 4);
  EB.oi.r_ctime = imm.alloc(n1 * 8); EB.oi.r_uid_rank = imm.alloc(n1 * 4); EB.oi.r_flags = imm.alloc(n1 * 4);
  EB.oi.pt_task = imm.alloc(T1 * 4); EB.oi.pt_off = imm.alloc(((size_t)J + 1) * 4);
  EB.oi.task_class = imm.alloc(T1 * 4); EB.oi.task_present = imm.alloc(T1 * 4); EB.oi.job_waiting0 = imm.alloc(J1 * 4);
  EB.oi.r_atom_off = imm.alloc(((size_t)n + 1) * 4); EB.oi.r_atom = imm.alloc(std::max<size_t>(1, r_atom.size()) * 4);
  EB.oi.atom_bit = imm.alloc(std::max(1u, NA) * 4); EB.oi.atom_local = imm.alloc(atom_local.size() * 4);
  EB.om.r_state = mut.alloc(n1); EB.om.pt_pos = mut.alloc(J1 * 4); EB.om.job_waiting = mut.alloc(J1 * 4);
  EB.om.jheap = mut.alloc(J1 * 4); EB.om.jheap_len = mut.alloc(Q1 * 4); EB.om.qheap = mut.alloc(Q1 * 4); EB.om.queue_map = mut.alloc(Q1 * 4);
  EB.om.q_alloc_present = mut.alloc(Q1 * 4); EB.om.evict_order = mut.alloc(n1 * 4);
  EB.om.ops = mut.alloc((n1 + T1) * 4); EB.om.scratch = mut.alloc((size_t)KB_EVICT_MAXV * 4); EB.om.ctl = mut.alloc(sizeof(EvictCtl));
  EB.om.atom_cnt = mut.alloc(std::max<size_t>(1, (size_t)NA * N) * 4);      // part of the pristine copy: every cycle starts from it
  imm.commit(); mut.commit();
  unsigned char* ib = imm.host.data(); unsigned char* mb = mut.host.data();
  uint32_t* node_off = (uint32_t*)(ib + EB.oi.node_off);
  for (uint32_t k = 0; k < n; ++k) node_off[run->node[order[k]] + 1] += 1;
  for (uint32_t i = 0; i < N; ++i) node_off[i + 1] += node_off[i];
  for (uint32_t k = 0; k < n; ++k) {
    const uint32_t i = order[k];
    ((uint32_t*)(ib + EB.oi.r_orig))[k] = i; ((uint32_t*)(ib + EB.oi.r_job))[k] = run->job[i];
    for (uint32_t r = 0; r < R; ++r) ((double*)(ib + EB.oi.r_resreq))[(size_t)r * n + k] = run->resreq[(size_t)r * n + i];
    ((uint32_t*)(ib + EB.oi.r_present))[k] = run->res_present[i]; ((int32_t*)(ib + EB.oi.r_prio))[k] = run->prio[i];
    ((int64_t*)(ib + EB.oi.r_ctime))[k] = run->ctime[i]; ((uint32_t*)(ib + EB.oi.r_uid_rank))[k] = run->uid_rank[i];
    ((uint32_t*)(ib + EB.oi.r_flags))[k] = run->flags[i];
  }
  if (T) {
    memcpy(ib + EB.oi.pt_task, pt.data(), (size_t)T * 4);
    memcpy(ib + EB.oi.task_class, B.imm.host.data() + B.oi.task_class, (size_t)T * 4);
    memcpy(ib + EB.oi.task_present, s->task_res_present, (size_t)T * 4);
  }
  memcpy(ib + EB.oi.pt_off, pt_off.data(), ((size_t)J + 1) * 4);
  if (lists) {
    memcpy(ib + EB.oi.r_atom_off, r_atom_off.data(), r_atom_off.size() * 4);
    if (!r_atom.empty()) memcpy(ib + EB.oi.r_atom, r_atom.data(), r_atom.size() * 4);
    if (NA) memcpy(ib + EB.oi.atom_bit, atom_bit.data(), (size_t)NA * 4);
  }
  memcpy(ib + EB.oi.atom_local, atom_local.data(), atom_local.size() * 4);
  // members per (atom, node) as loaded: the group's counter of the node's domain (an atom's key set has one domain per node)
  if (NA) {
    std::vector<uint32_t> gbase(NG + 1, 0);
    for (uint32_t g = 0; g < NG; ++g) gbase[g + 1] = gbase[g] + pa->keyset_domains[pa->group_keyset[g]];
    std::vector<int32_t> group_of_atom((size_t)64 * B.W, -1);
    for (uint32_t g = 0; g < NG; ++g) if (B.aff_atom_of_group[g] >= 0) group_of_atom[B.aff_atom_of_group[g]] = (int32_t)g;
    int32_t* cnt = (int32_t*)(mb + EB.om.atom_cnt);
    for (uint32_t l = 0; l < NA; ++l) {
      const uint32_t g = (uint32_t)group_of_atom[atom_bit[l]], ks = pa->group_keyset[g];
      for (uint32_t v = 0; v < N; ++v) cnt[(size_t)l * N + v] = pa->group_count0[gbase[g] + (uint32_t)pa->node_domain[(size_t)ks * N + v]];
    }
  }
  // ---- mutable state as the actions find it ----
  uint32_t* evo = (uint32_t*)(mb + EB.om.evict_order);
  for (uint32_t k = 0; k < n1; ++k) evo[k] = 0xFFFFFFFFu;
  int32_t* jw0 = (int32_t*)(ib + EB.oi.job_waiting0);
  for (uint32_t j = 0; j < J; ++j) jw0[j] = (run && run->job_waiting0) ? run->job_waiting0[j] : 0;
  for (uint32_t q = 0; q < Q; ++q) ((uint32_t*)(mb + EB.om.q_alloc_present))[q] = q < B.q_alloc_present.size() ? B.q_alloc_present[q] : 0u;
  // the actions' own queues (preemptorsMap, queues) are filled at the start of each action, on the state it finds: evict_init
  (void)H;
  return KB_OK;
}

}  // namespace kb
#endif  // KB_EVICT_BUILD_H_
