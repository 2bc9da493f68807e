// affinity_run.cpp — cluster objects with node affinity and inter-pod (anti)affinity through the C++ host mirror
// (kube_batch_b200/host/kbhost.hpp).  tests/test_host_cpp_affinity.py writes the file from the same objects it hands to
// kube_batch_b200/builder.py and compares the output with builder.py's tables and with the oracle.
//
//   affinity_run FILE          every `case` of FILE on a fresh cache + session, through the Cycle shells (mode "cycle") or the
//                              per-action allocate / backfill shells (mode "shells"): binds, evictions in call order, every node's
//                              Idle / Releasing / Used, every task's status — the output of tests/host/cycle_run
//   affinity_run --flat FILE   the session's flattening as one JSON object: the node-affinity relations of every (task, node),
//                              kb_snapshot.flags, the task flags, kb_pod_affinity and the Running table's affinity groups; no GPU
//
// Input: the lines of cycle_run (queue, node, podgroup, pod, case, tier, plugin; a case line takes a third word, the mode), plus
// lines that extend the object declared last ("-" is an empty string, VALUES a comma-separated list, "-" for none):
//   label KEY VALUE                     node or pod label
//   taint KEY VALUE EFFECT              node
//   toleration KEY OPERATOR VALUE EFFECT, selector KEY VALUE (nodeSelector), hostport IP PROTOCOL PORT      pod
//   required                            pod: a non-nil requiredDuringScheduling node selector (no terms yet)
//   term                                a NodeSelectorTerm of it
//   preferred WEIGHT                    a PreferredSchedulingTerm
//   expr KEY OPERATOR VALUES            a MatchExpression of the term started last (required term or preferred term)
//   field KEY OPERATOR VALUES           a MatchFields requirement of the required term started last
//   podaff aff|anti                     pod: a non-nil PodAffinity / PodAntiAffinity (no terms yet)
//   podterm aff|anti req|WEIGHT TOPOLOGYKEY NAMESPACES nil|sel      a required or weighted preferred PodAffinityTerm
//   matchlabel KEY VALUE, matchexpr KEY OPERATOR VALUES             its label selector
//   allocate NS NAME NODE               after the session opens: ssn.Allocate of that pending task (its Spec.NodeName stays "")
// Exit code: 0 done, 1 bad input or a refused session, 3 no CUDA device (the engine has no CPU fallback).
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iostream>
#include <sstream>

#include "../../kube_batch_b200/host/kbhost.hpp"

using namespace kb;

struct Case {
  std::string label, mode;
  std::vector<std::string> actions;
  std::vector<conf::Tier> tiers;
};

struct Cluster {
  struct Queue { std::string name; int weight; int64_t ctime; };
  struct Place { std::string ns, name, node; };
  std::vector<Queue> queues;
  std::vector<api::Node> nodes;
  std::vector<cache::PodGroup> podGroups;
  std::vector<api::Pod> pods;
  std::vector<Place> places;
  std::vector<Case> cases;
};

static std::string str(const std::string& s) { return s == "-" ? std::string() : s; }

static std::vector<std::string> list(const std::string& s) {
  std::vector<std::string> out;
  if (s == "-") return out;
  std::istringstream in(s);
  std::string v;
  while (std::getline(in, v, ',')) out.push_back(v);
  return out;
}

static void resources(std::istringstream& in, api::ResourceList& rl) {
  std::string kv;
  while (in >> kv) {
    size_t eq = kv.find('=');
    if (eq == std::string::npos) throw std::runtime_error("bad resource " + kv);
    rl[kv.substr(0, eq)] = std::stod(kv.substr(eq + 1));
  }
}

static Cluster parse(const char* path) {
  std::ifstream f(path);
  if (!f) throw std::runtime_error(std::string("cannot read ") + path);
  Cluster c;
  std::string line;
  bool lastIsNode = false;
  char nodeTerm = 0;                                  // 'r': the last required term, 'p': the last preferred term
  api::PodAffinityTerm* podTerm = nullptr;
  auto pod = [&]() -> api::Pod& { if (c.pods.empty() || lastIsNode) throw std::runtime_error("no pod for: " + line); return c.pods.back(); };
  auto affinity = [&]() -> api::Affinity& { auto& p = pod(); if (!p.Affinity) p.Affinity = std::make_shared<api::Affinity>(); return *p.Affinity; };
  auto nodeAffinity = [&]() -> api::NodeAffinity& { auto& a = affinity(); if (!a.NodeAffinity) a.NodeAffinity = std::make_shared<api::NodeAffinity>(); return *a.NodeAffinity; };
  auto podAffinity = [&](const std::string& kind) -> api::PodAffinity& {
    if (kind != "aff" && kind != "anti") throw std::runtime_error("bad line: " + line);
    auto& a = affinity();
    auto& pa = kind == "aff" ? a.PodAffinity : a.PodAntiAffinity;
    if (!pa) pa = std::make_shared<api::PodAffinity>();
    return *pa;
  };
  while (std::getline(f, line)) {
    std::istringstream in(line);
    std::string kind;
    if (!(in >> kind)) continue;
    if (kind == "queue") {
      std::string name; int weight; int64_t ctime;
      in >> name >> weight >> ctime;
      c.queues.push_back({name, weight, ctime});
    } else if (kind == "node") {
      api::Node n; in >> n.Name; resources(in, n.Allocatable); c.nodes.push_back(n); lastIsNode = true;
    } else if (kind == "podgroup") {
      cache::PodGroup pg; in >> pg.Namespace >> pg.Name >> pg.Queue >> pg.MinMember >> pg.Priority >> pg.CreationTimestamp; c.podGroups.push_back(pg);
    } else if (kind == "pod") {
      api::Pod p; int deleting = 0;
      in >> p.Namespace >> p.Name >> p.UID >> p.NodeName >> p.Phase >> deleting >> p.Priority >> p.CreationTimestamp >> p.GroupName >> p.PriorityClassName;
      p.NodeName = str(p.NodeName); p.PriorityClassName = str(p.PriorityClassName); p.Deleting = deleting != 0;
      resources(in, p.Requests);
      c.pods.push_back(p); lastIsNode = false; nodeTerm = 0; podTerm = nullptr;
    } else if (kind == "label") {
      std::string k, v; in >> k >> v;
      if (lastIsNode && !c.nodes.empty()) c.nodes.back().Labels[k] = str(v); else pod().Labels[k] = str(v);
    } else if (kind == "taint") {
      if (!lastIsNode || c.nodes.empty()) throw std::runtime_error("taint without a node");
      api::Node::Taint t; in >> t.Key >> t.Value >> t.Effect; t.Value = str(t.Value); c.nodes.back().Taints.push_back(t);
    } else if (kind == "toleration") {
      api::Pod::Toleration t; in >> t.Key >> t.Operator >> t.Value >> t.Effect;
      t.Key = str(t.Key); t.Operator = str(t.Operator); t.Value = str(t.Value); t.Effect = str(t.Effect);
      pod().Tolerations.push_back(t);
    } else if (kind == "selector") {
      std::string k, v; in >> k >> v; pod().NodeSelector[k] = str(v);
    } else if (kind == "hostport") {
      api::Pod::HostPort h; in >> h.HostIP >> h.Protocol >> h.Port; h.HostIP = str(h.HostIP); h.Protocol = str(h.Protocol); pod().HostPorts.push_back(h);
    } else if (kind == "required") {
      nodeAffinity().RequiredDuringSchedulingIgnoredDuringExecution = std::make_shared<api::NodeSelector>();
    } else if (kind == "term") {
      auto& req = nodeAffinity().RequiredDuringSchedulingIgnoredDuringExecution;
      if (!req) throw std::runtime_error("term before required");
      req->NodeSelectorTerms.emplace_back(); nodeTerm = 'r';
    } else if (kind == "preferred") {
      api::PreferredSchedulingTerm t; in >> t.Weight;
      nodeAffinity().PreferredDuringSchedulingIgnoredDuringExecution.push_back(t); nodeTerm = 'p';
    } else if (kind == "expr" || kind == "field") {
      api::NodeSelectorRequirement r; std::string vals; in >> r.Key >> r.Operator >> vals; r.Values = list(vals);
      auto& na = nodeAffinity();
      if (nodeTerm == 'r') {
        auto& t = na.RequiredDuringSchedulingIgnoredDuringExecution->NodeSelectorTerms.back();
        (kind == "expr" ? t.MatchExpressions : t.MatchFields).push_back(r);
      } else if (nodeTerm == 'p' && kind == "expr") {
        na.PreferredDuringSchedulingIgnoredDuringExecution.back().Preference.MatchExpressions.push_back(r);
      } else {
        throw std::runtime_error("no node-selector term for: " + line);
      }
    } else if (kind == "podaff") {
      std::string k; in >> k; podAffinity(k);
    } else if (kind == "podterm") {
      std::string k, w, topo, ns, sel; in >> k >> w >> topo >> ns >> sel;
      api::PodAffinityTerm t; t.TopologyKey = str(topo); t.Namespaces = list(ns);
      if (sel == "sel") t.LabelSelector = std::make_shared<api::LabelSelector>();
      else if (sel != "nil") throw std::runtime_error("bad selector in: " + line);
      auto& pa = podAffinity(k);
      if (w == "req") { pa.RequiredDuringSchedulingIgnoredDuringExecution.push_back(t); podTerm = &pa.RequiredDuringSchedulingIgnoredDuringExecution.back(); }
      else { pa.PreferredDuringSchedulingIgnoredDuringExecution.push_back({std::stoi(w), t}); podTerm = &pa.PreferredDuringSchedulingIgnoredDuringExecution.back().PodAffinityTerm; }
    } else if (kind == "matchlabel" || kind == "matchexpr") {
      if (!podTerm || !podTerm->LabelSelector) throw std::runtime_error("no pod affinity term with a selector for: " + line);
      if (kind == "matchlabel") { std::string k, v; in >> k >> v; podTerm->LabelSelector->MatchLabels[k] = str(v); }
      else { api::LabelSelectorRequirement r; std::string vals; in >> r.Key >> r.Operator >> vals; r.Values = list(vals); podTerm->LabelSelector->MatchExpressions.push_back(r); }
    } else if (kind == "allocate") {
      Cluster::Place pl; in >> pl.ns >> pl.name >> pl.node; c.places.push_back(pl);
    } else if (kind == "case") {
      Case k; std::string acts; in >> k.label >> acts >> k.mode;
      if (k.mode != "cycle" && k.mode != "shells") throw std::runtime_error("case mode must be cycle or shells: " + line);
      std::istringstream a(acts); std::string name;
      while (std::getline(a, name, ',')) k.actions.push_back(name);
      c.cases.push_back(k);
    } else if (kind == "tier") {
      if (c.cases.empty()) throw std::runtime_error("tier before case");
      c.cases.back().tiers.emplace_back();
    } else if (kind == "plugin") {
      if (c.cases.empty() || c.cases.back().tiers.empty()) throw std::runtime_error("plugin before tier");
      conf::PluginOption o; in >> o.Name;
      for (int* e : {&o.EnabledJobOrder, &o.EnabledJobReady, &o.EnabledJobPipelined, &o.EnabledTaskOrder, &o.EnabledPreemptable,
                     &o.EnabledReclaimable, &o.EnabledQueueOrder, &o.EnabledPredicate, &o.EnabledNodeOrder}) in >> *e;
      std::string kv;
      while (in >> kv) { size_t eq = kv.find('='); o.Arguments[kv.substr(0, eq)] = kv.substr(eq + 1); }
      c.cases.back().tiers.back().Plugins.push_back(o);
    } else {
      throw std::runtime_error("unknown line: " + line);
    }
    if (in.fail() && !in.eof()) throw std::runtime_error("bad line: " + line);
  }
  return c;
}

static std::unique_ptr<framework::Session> open(cache::SchedulerCache& sc, const Cluster& c, const std::vector<conf::Tier>& tiers) {
  for (auto& n : c.nodes) sc.AddNode(n);
  for (auto& p : c.pods) sc.AddPod(p);
  for (auto& pg : c.podGroups) sc.AddPodGroup(pg);
  for (auto& q : c.queues) { sc.AddQueue(q.name, q.weight); sc.Queues[q.name]->CreationTimestamp = q.ctime; }
  auto ssn = framework::OpenSession(&sc, tiers);
  for (auto& pl : c.places) {
    std::shared_ptr<api::TaskInfo> task;
    for (auto& jk : ssn->Jobs) for (auto& tk : jk.second->Tasks) if (tk.second->Namespace == pl.ns && tk.second->Name == pl.name) task = tk.second;
    if (!task) throw std::runtime_error("allocate: no task " + pl.ns + "/" + pl.name);
    ssn->Allocate(task, pl.node);
  }
  return ssn;
}

// ------------------------------------------------------------------------------------------------------------- --flat
template <class V> static void arr(const char* name, const V& v, size_t n, bool comma = true) {
  printf("\"%s\": [", name);
  for (size_t i = 0; i < n; ++i) printf("%s%lld", i ? ", " : "", (long long)v[i]);
  printf("]%s\n", comma ? "," : "");
}

static void names(const char* name, const std::vector<std::string>& v) {
  printf("\"%s\": [", name);
  for (size_t i = 0; i < v.size(); ++i) printf("%s\"%s\"", i ? ", " : "", v[i].c_str());
  printf("],\n");
}

static int dumpFlat(const Cluster& c) {
  cache::SchedulerCache sc;
  auto ssn = open(sc, c, {});
  actions::allocate::Flat f = actions::allocate::Flatten(*ssn);
  actions::cycle::Running r = actions::cycle::FlattenRunning(*ssn, f);
  const uint32_t N = f.N, T = f.T, W = f.W;
  printf("{\n");
  names("nodes", f.nodeNames);
  std::vector<std::string> tasks;
  for (auto& t : f.tasks) tasks.push_back(t->Namespace + "/" + t->Name);
  names("tasks", tasks);
  printf("\"W\": %u, \"flags\": %u,\n", W, f.snap_flags);
  arr("task_flags", f.task_flags, T);
  arr("task_n_aff", f.task_n_aff, T);
  arr("task_n_pref", f.task_n_pref, T);
  // the relations the atoms encode: required node affinity matches (OR over the terms of an AND of atoms), preferred count
  printf("\"aff_match\": [");
  for (uint32_t t = 0; t < T; ++t) {
    printf("%s[", t ? ", " : "");
    for (uint32_t n = 0; n < N; ++n) {
      bool ok = f.task_n_aff[t] == 0;
      for (uint32_t k = 0; k < f.task_n_aff[t] && !ok; ++k) {
        bool all = true;
        for (uint32_t w = 0; w < W; ++w) { uint64_t need = f.task_aff[((size_t)k * W + w) * T + t]; all = all && (f.node_labels[(size_t)w * N + n] & need) == need; }
        ok = all;
      }
      printf("%s%d", n ? ", " : "", ok ? 1 : 0);
    }
    printf("]");
  }
  printf("],\n\"pref_count\": [");
  for (uint32_t t = 0; t < T; ++t) {
    printf("%s[", t ? ", " : "");
    for (uint32_t n = 0; n < N; ++n) {
      long long cnt = 0;
      for (uint32_t k = 0; k < f.task_n_pref[t]; ++k) {
        bool all = true;
        for (uint32_t w = 0; w < W; ++w) { uint64_t need = f.task_pref[((size_t)k * W + w) * T + t]; all = all && (f.node_labels[(size_t)w * N + n] & need) == need; }
        if (all) cnt += f.task_pref_w[(size_t)k * T + t];
      }
      printf("%s%lld", n ? ", " : "", cnt);
    }
    printf("]");
  }
  printf("],\n");
  // the Running table's affinity part
  const size_t n = r.tasks.size();
  std::vector<std::string> rnames;
  for (auto& t : r.tasks) rnames.push_back(t->Namespace + "/" + t->Name);
  names("running", rnames);
  arr("running_flags", r.flags, n);
  arr("running_aff_group_off", r.aff_group_off, n + 1);
  arr("running_aff_group", r.aff_group, r.aff_group_off[n]);
  const auto& pa = f.pa;
  if (!pa.on) { printf("\"pod_affinity\": null\n}\n"); return 0; }
  const uint32_t NG = pa.n_groups, NK = pa.n_kinds;
  printf("\"pod_affinity\": {\n\"n_keysets\": %u, \"n_groups\": %u, \"n_kinds\": %u, \"first_unbound_node\": %d,\n", pa.n_keysets, NG, NK, pa.first_unbound);
  arr("node_domain", pa.node_domain, (size_t)pa.n_keysets * N);
  arr("keyset_domains", pa.keyset_domains, pa.n_keysets);
  arr("group_keyset", pa.group_keyset, NG);
  size_t ncount = 0;
  for (uint32_t g = 0; g < NG; ++g) ncount += pa.keyset_domains[pa.group_keyset[g]];
  arr("group_count0", pa.group_count0, ncount);
  arr("group_total0", pa.group_total0, NG);
  printf("\"task_forbid\": [");                       // unsigned 64-bit masks as strings (JSON numbers lose them)
  for (uint32_t t = 0; t < T; ++t) printf("%s\"%llu\"", t ? ", " : "", (unsigned long long)pa.task_forbid[t]);
  printf("],\n\"task_contrib\": [");
  for (uint32_t t = 0; t < T; ++t) printf("%s\"%llu\"", t ? ", " : "", (unsigned long long)pa.task_contrib[t]);
  printf("],\n");
  arr("task_need", pa.task_need, T);
  arr("task_kind", pa.task_kind, T);
  arr("node_kind_count0", pa.node_kind_count0, (size_t)NK * N);
  arr("kind_unbound", pa.kind_unbound, NK);
  arr("task_weight_off", pa.task_weight_off, T + 1);
  const size_t nw = pa.task_weight_off[T];
  arr("weight_kind", pa.weight_kind, nw);
  arr("weight_keyset", pa.weight_keyset, nw);
  arr("weight_value", pa.weight_value, nw);
  if (!pa.task_xgroup_off.empty()) {
    arr("task_xgroup_off", pa.task_xgroup_off, T + 1);
    arr("task_xgroup", pa.task_xgroup, pa.task_xgroup_off[T]);
  }
  printf("\"end\": 0\n}\n}\n");
  framework::CloseSession(ssn.get());
  return 0;
}

// ------------------------------------------------------------------------------------------------------------- cases
static void printResource(const char* what, const api::Resource& r) {
  printf(" %s cpu=%.17g memory=%.17g", what, r.MilliCPU, r.Memory);
  for (auto& kv : r.ScalarResources) printf(" %s=%.17g", kv.first.c_str(), kv.second);
}

int main(int argc, char** argv) {
  const bool flat = argc == 3 && !strcmp(argv[1], "--flat");
  if (argc != 2 && !flat) { fprintf(stderr, "usage: affinity_run [--flat] FILE\n"); return 1; }
  plugins::RegisterBuiltins();
  Cluster c;
  try { c = parse(argv[argc - 1]); } catch (const std::exception& e) { fprintf(stderr, "%s\n", e.what()); return 1; }
  if (flat) {
    try { return dumpFlat(c); } catch (const std::exception& e) { fprintf(stderr, "error %s\n", e.what()); return 1; }
  }
  int rc = 0;
  for (auto& k : c.cases) {
    auto binder = std::make_shared<cache::FakeBinder>();
    auto evictor = std::make_shared<cache::FakeEvictor>();
    cache::SchedulerCache sc;
    sc.binder = binder;
    sc.evictor = evictor;
    auto ssn = open(sc, c, k.tiers);
    printf("case %s\n", k.label.c_str());
    try {
      if (k.mode == "cycle") {
        auto cycle = actions::cycle::New(k.actions);
        auto shells = cycle->Actions();
        for (auto& name : k.actions)                    // scheduler.go:88-92: the configured actions, in order, on one session
          for (auto& a : shells) if (a->Name() == name) a->Execute(ssn.get());
      } else {
        for (auto& name : k.actions) {                  // one flatten + kb_allocate / kb_backfill per action
          if (name == "allocate") actions::allocate::New()->Execute(ssn.get());
          else if (name == "backfill") actions::backfill::New()->Execute(ssn.get());
          else throw std::runtime_error("the per-action shells are allocate and backfill, not " + name);
        }
      }
    } catch (const std::exception& e) {
      printf("error %s\nend\n", e.what());
      fflush(stdout);
      fprintf(stderr, "case %s: %s\n", k.label.c_str(), e.what());
      framework::CloseSession(ssn.get());
      if (strstr(e.what(), "KB_E_CUDA")) return 3;
      rc = 1;
      continue;
    }
    framework::CloseSession(ssn.get());
    for (auto& kv : binder->Binds) printf("bind %s %s\n", kv.first.c_str(), kv.second.c_str());
    for (auto& e : evictor->Evicts) printf("evict %s\n", e.c_str());
    for (auto& kv : ssn->Nodes) {
      printf("node %s", kv.first.c_str());
      printResource("idle", kv.second->Idle); printResource("releasing", kv.second->Releasing); printResource("used", kv.second->Used);
      printf("\n");
    }
    for (auto& jk : ssn->Jobs) for (auto& tk : jk.second->Tasks) printf("task %s/%s %d\n", tk.second->Namespace.c_str(), tk.second->Name.c_str(), tk.second->Status);
    printf("end\n");
  }
  return rc;
}
