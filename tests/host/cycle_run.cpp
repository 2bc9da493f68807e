// cycle_run.cpp — runs action lists through the C++ host mirror's cycle shells (kb::actions::cycle) on cluster objects read
// from a line-oriented text file, and prints what the cache saw.  tests/test_host_cpp_cycle.py writes the file from the same
// objects it hands to kube_batch_b200/builder.py and compares the output with the oracle.
//
//   cycle_run FILE            every `case` of FILE on a fresh cache + session: binds (FakeBinder), evictions in call order
//                             (FakeEvictor), every node's Idle / Releasing / Used, every task's status
//   cycle_run --running FILE  the session's flattened Running table (FlattenRunning) and job_waiting0; host code, no GPU
//
// Input, one object per line, whitespace-separated; "-" is an empty string; resources are name=quantity (cpu in cores,
// memory in bytes, pods, scalars in units):
//   queue NAME WEIGHT CTIME
//   node NAME RES...
//   podgroup NS NAME QUEUE MINMEMBER PRIORITY CTIME
//   pod NS NAME UID NODE PHASE DELETING PRIORITY CTIME GROUP PRIORITYCLASS RES...
//   case LABEL ACTION[,ACTION...]                  then its tiers:
//   tier                                           starts a tier
//   plugin NAME JOBORDER JOBREADY JOBPIPELINED TASKORDER PREEMPTABLE RECLAIMABLE QUEUEORDER PREDICATE NODEORDER [KEY=VALUE...]
//                                                  (-1 nil, 0 false, 1 true)
// Output lines: "case LABEL", "bind TASK NODE", "evict TASK", "node NAME idle|releasing|used RES...", "task TASK STATUS",
// "end"; "error MESSAGE" when the engine refuses the session.
// Exit code: 0 done, 1 bad input or a refused session, 3 no CUDA device (the engine has no CPU fallback).
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iostream>
#include <sstream>

#include "../../kube_batch_b200/host/kbhost.hpp"

using namespace kb;

struct Case {
  std::string label;
  std::vector<std::string> actions;
  std::vector<conf::Tier> tiers;
};

struct Cluster {
  struct Queue { std::string name; int weight; int64_t ctime; };
  std::vector<Queue> queues;
  std::vector<api::Node> nodes;
  std::vector<cache::PodGroup> podGroups;
  std::vector<api::Pod> pods;
  std::vector<Case> cases;
};

static std::string str(const std::string& s) { return s == "-" ? std::string() : s; }

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
  while (std::getline(f, line)) {
    std::istringstream in(line);
    std::string kind;
    if (!(in >> kind)) continue;
    if (kind == "queue") {
      std::string name; int weight; int64_t ctime;
      in >> name >> weight >> ctime;
      c.queues.push_back({name, weight, ctime});
    } else if (kind == "node") {
      api::Node n; in >> n.Name; resources(in, n.Allocatable); c.nodes.push_back(n);
    } else if (kind == "podgroup") {
      cache::PodGroup pg; in >> pg.Namespace >> pg.Name >> pg.Queue >> pg.MinMember >> pg.Priority >> pg.CreationTimestamp; c.podGroups.push_back(pg);
    } else if (kind == "pod") {
      api::Pod p; int deleting = 0;
      in >> p.Namespace >> p.Name >> p.UID >> p.NodeName >> p.Phase >> deleting >> p.Priority >> p.CreationTimestamp >> p.GroupName >> p.PriorityClassName;
      p.NodeName = str(p.NodeName); p.PriorityClassName = str(p.PriorityClassName); p.Deleting = deleting != 0;
      resources(in, p.Requests);
      c.pods.push_back(p);
    } else if (kind == "case") {
      Case k; std::string acts; in >> k.label >> acts;
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

static void fill(cache::SchedulerCache& sc, const Cluster& c) {
  for (auto& n : c.nodes) sc.AddNode(n);
  for (auto& p : c.pods) sc.AddPod(p);
  for (auto& pg : c.podGroups) sc.AddPodGroup(pg);
  for (auto& q : c.queues) { sc.AddQueue(q.name, q.weight); sc.Queues[q.name]->CreationTimestamp = q.ctime; }
}

static void printResource(const char* what, const api::Resource& r) {
  printf(" %s cpu=%.17g memory=%.17g", what, r.MilliCPU, r.Memory);
  for (auto& kv : r.ScalarResources) printf(" %s=%.17g", kv.first.c_str(), kv.second);
}

static int dumpRunning(const Cluster& c) {
  cache::SchedulerCache sc;
  fill(sc, c);
  auto ssn = framework::OpenSession(&sc, {});
  actions::allocate::Flat f = actions::allocate::Flatten(*ssn);
  actions::cycle::Running r = actions::cycle::FlattenRunning(*ssn, f);
  const size_t n = r.tasks.size();
  printf("dims");
  for (auto& d : f.dims) printf(" %s", d.c_str());
  printf("\n");
  for (size_t i = 0; i < n; ++i) {
    auto& t = *r.tasks[i];
    printf("running %s/%s %u %u %u %u %u %d %lld", t.Namespace.c_str(), t.Name.c_str(), r.node[i], r.job[i], r.present[i], r.uid_rank[i], r.flags[i],
           r.prio[i], (long long)r.ctime[i]);
    for (uint32_t k = 0; k < f.R; ++k) printf(" %.17g", r.resreq[k * n + i]);
    printf("\n");
  }
  printf("waiting");
  for (size_t j = 0; j < f.jobIDs.size(); ++j) printf(" %d", r.waiting[j]);
  printf("\n");
  framework::CloseSession(ssn.get());
  return 0;
}

int main(int argc, char** argv) {
  const bool running = argc == 3 && !strcmp(argv[1], "--running");
  if (argc != 2 && !running) { fprintf(stderr, "usage: cycle_run [--running] FILE\n"); return 1; }
  plugins::RegisterBuiltins();
  Cluster c;
  try { c = parse(argv[argc - 1]); } catch (const std::exception& e) { fprintf(stderr, "%s\n", e.what()); return 1; }
  if (running) return dumpRunning(c);
  int rc = 0;
  for (auto& k : c.cases) {
    auto binder = std::make_shared<cache::FakeBinder>();
    auto evictor = std::make_shared<cache::FakeEvictor>();
    cache::SchedulerCache sc;
    sc.binder = binder;
    sc.evictor = evictor;
    fill(sc, c);
    auto ssn = framework::OpenSession(&sc, k.tiers);
    printf("case %s\n", k.label.c_str());
    try {
      auto cycle = actions::cycle::New(k.actions);
      auto shells = cycle->Actions();
      for (auto& name : k.actions)                      // scheduler.go:88-92: the configured actions, in order, on one session
        for (auto& a : shells) if (a->Name() == name) a->Execute(ssn.get());
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
