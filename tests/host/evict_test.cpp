// evict_test.cpp — the reference's preempt and reclaim action tests, restated against the C++ host mirror + libkbgpu.so.
// Mirrors kube-batch/pkg/scheduler/actions/preempt/preempt_test.go:37-202 and actions/reclaim/reclaim_test.go:37-170 (same objects,
// same tiers, same expected number of FakeEvictor.Evict calls).  The action runs through the cycle shells
// (kb::actions::cycle), i.e. kb_session_load_running + kb_cycle and the replay through Session::Evict / Statement.
// Exit code: 0 all cases passed, 1 a case failed, 3 no CUDA device (the engine has no CPU fallback).
#include <cstring>
#include <iostream>

#include "../../kube_batch_b200/host/kbhost.hpp"

using namespace kb;

static api::ResourceList BuildResourceList(double cpu, double memory) { return {{"cpu", cpu}, {"memory", memory}, {"nvidia.com/gpu", 0}}; }   // util/test_utils.go:34-40
static api::Node BuildNode(const std::string& name, api::ResourceList alloc) { api::Node n; n.Name = name; n.Allocatable = std::move(alloc); return n; }
static api::Pod BuildPod(const std::string& ns, const std::string& name, const std::string& node, const std::string& phase,
                         api::ResourceList req, const std::string& group) {
  api::Pod p; p.Namespace = ns; p.Name = name; p.UID = ns + "-" + name; p.NodeName = node; p.Phase = phase; p.Requests = std::move(req); p.GroupName = group; return p;
}

struct Case {
  std::string name, action;
  std::vector<cache::PodGroup> podGroups;
  std::vector<api::Pod> pods;
  std::vector<api::Node> nodes;
  std::vector<std::string> queues;
  int expected;
};

int main() {
  const double G = 1e9, Gi = 1024.0 * 1024.0 * 1024.0;
  plugins::RegisterBuiltins();                          // framework.RegisterPluginBuilder("conformance" / "gang", ...)
  const api::ResourceList r1 = BuildResourceList(1, 1 * G);

  std::vector<Case> tests;
  tests.push_back({"preempt: one Job with two Pods on one node", "preempt",                                  // preempt_test.go:49-83
                   {{"c1", "pg1", "q1"}},
                   {BuildPod("c1", "preemptee1", "n1", "Running", r1, "pg1"), BuildPod("c1", "preemptee2", "n1", "Running", r1, "pg1"),
                    BuildPod("c1", "preemptor1", "", "Pending", r1, "pg1"), BuildPod("c1", "preemptor2", "", "Pending", r1, "pg1")},
                   {BuildNode("n1", BuildResourceList(3, 3 * Gi))}, {"q1"}, 1});
  tests.push_back({"preempt: two Jobs on one node", "preempt",                                               // preempt_test.go:84-131
                   {{"c1", "pg1", "q1"}, {"c1", "pg2", "q1"}},
                   {BuildPod("c1", "preemptee1", "n1", "Running", r1, "pg1"), BuildPod("c1", "preemptee2", "n1", "Running", r1, "pg1"),
                    BuildPod("c1", "preemptor1", "", "Pending", r1, "pg2"), BuildPod("c1", "preemptor2", "", "Pending", r1, "pg2")},
                   {BuildNode("n1", BuildResourceList(2, 2 * G))}, {"q1"}, 2});
  tests.push_back({"reclaim: two Queues with one Job each", "reclaim",                                       // reclaim_test.go:50-100
                   {{"c1", "pg1", "q1"}, {"c1", "pg2", "q2"}},
                   {BuildPod("c1", "preemptee1", "n1", "Running", r1, "pg1"), BuildPod("c1", "preemptee2", "n1", "Running", r1, "pg1"),
                    BuildPod("c1", "preemptee3", "n1", "Running", r1, "pg1"), BuildPod("c1", "preemptor1", "", "Pending", r1, "pg2")},
                   {BuildNode("n1", BuildResourceList(3, 3 * Gi))}, {"q1", "q2"}, 1});

  int failed = 0;
  for (size_t i = 0; i < tests.size(); ++i) {
    auto& test = tests[i];
    auto binder = std::make_shared<cache::FakeBinder>();
    auto evictor = std::make_shared<cache::FakeEvictor>();
    cache::SchedulerCache schedulerCache;
    schedulerCache.binder = binder;
    schedulerCache.evictor = evictor;
    for (auto& node : test.nodes) schedulerCache.AddNode(node);
    for (auto& pod : test.pods) schedulerCache.AddPod(pod);
    for (auto& ss : test.podGroups) schedulerCache.AddPodGroup(ss);
    for (auto& q : test.queues) schedulerCache.AddQueue(q, 1);
    // conformance + gang with EnabledPreemptable (preempt_test.go:171-186) / EnabledReclaimable (reclaim_test.go:140-154)
    conf::PluginOption conformance; conformance.Name = "conformance";
    conf::PluginOption gang; gang.Name = "gang";
    if (test.action == "preempt") conformance.EnabledPreemptable = gang.EnabledPreemptable = 1;
    else conformance.EnabledReclaimable = gang.EnabledReclaimable = 1;
    auto ssn = framework::OpenSession(&schedulerCache, {conf::Tier{{conformance, gang}}});
    try {
      auto shells = actions::cycle::New({test.action})->Actions();
      for (auto& a : shells) if (a->Name() == test.action) a->Execute(ssn.get());
    } catch (const std::exception& e) {
      std::cerr << "case " << i << " (" << test.name << "): Execute failed loudly: " << e.what() << "\n";
      framework::CloseSession(ssn.get());
      return strstr(e.what(), "KB_E_CUDA") ? 3 : 1;
    }
    framework::CloseSession(ssn.get());
    if ((int)evictor->Evicts.size() != test.expected) {
      ++failed;
      std::cerr << "case " << i << " (" << test.name << "): expected " << test.expected << " evictions, got " << evictor->Evicts.size() << "\n";
    } else {
      std::cout << "ok   case " << i << " (" << test.name << "): " << evictor->Evicts.size() << " eviction(s)\n";
    }
  }
  return failed ? 1 : 0;
}
