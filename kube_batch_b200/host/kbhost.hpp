// kbhost.hpp — C++17 host-side mirror of the kube-batch interface around the scheduling actions, sitting ABOVE the
// C ABI of libkbgpu.so (include/kbgpu.h).  The reference is Go and no Go toolchain exists in this image, so this
// header plays the role the Go shim (go/kbgpu) plays inside kube-batch: same names, same argument meaning, same
// error behaviour, so tests can be written like pkg/scheduler/actions/{allocate,preempt,reclaim}/*_test.go.
//
//   kb::api        Resource, TaskInfo, NodeInfo, JobInfo, QueueInfo, TaskStatus      (pkg/scheduler/api)
//   kb::conf       PluginOption, Tier                                                 (pkg/scheduler/conf)
//   kb::cache      SchedulerCache{AddNode,AddPod,AddPodGroup,AddQueue,Snapshot,Evict}, Binder, Evictor (pkg/scheduler/cache)
//   kb::framework  Session, Statement, Plugin, Action, Arguments, RegisterPluginBuilder, OpenSession, CloseSession
//   kb::plugins    the built-in plugin builders by name                                (pkg/scheduler/plugins/factory.go)
//   kb::actions::allocate::New()->Execute(ssn)                                         (pkg/scheduler/actions/allocate)
//   kb::actions::cycle::Cycle  the whole action list as ONE kb_cycle, replayed by four action shells (go/kbgpu/cycle.go)
//
// What differs from the reference, by construction: plugin callbacks are arbitrary Go closures there; a GPU engine
// can only honour the BUILT-IN ones.  Session::Add*Fn therefore registers a *descriptor* (which built-in function,
// from which plugin); Execute refuses loudly (std::runtime_error) when a tier names a plugin that registered a
// foreign function.  There is NO CPU fallback: Execute without a CUDA device throws.
#pragma once

#include <algorithm>
#include <cerrno>
#include <cmath>
#include <cstdlib>
#include <cstdint>
#include <functional>
#include <map>
#include <memory>
#include <set>
#include <stdexcept>
#include <string>
#include <tuple>
#include <vector>

#include "../../include/kbgpu.h"
#include "../csrc/kb_core.h"      // KB_NARROW_R / KB_NARROW_W: the capacities no kernel instance exceeds both of

namespace kb {

// ------------------------------------------------------------------------------------------------- api
namespace api {

using ResourceList = std::map<std::string, double>;   // v1.ResourceList: "cpu" cores, "memory" bytes, "pods", scalars in units

struct Resource {                                     // api/resource_info.go:28-38
  double MilliCPU = 0, Memory = 0;
  std::map<std::string, double> ScalarResources;      // empty == nil
  int MaxTaskNum = 0;
  static Resource New(const ResourceList& rl) {       // NewResource, resource_info.go:73-90
    Resource r;
    for (auto& kv : rl) {
      if (kv.first == "cpu") r.MilliCPU += std::ceil(kv.second * 1000.0 - 1e-9);      // Quantity.MilliValue rounds up
      else if (kv.first == "memory") r.Memory += kv.second;
      else if (kv.first == "pods") r.MaxTaskNum += (int)kv.second;
      else r.ScalarResources[kv.first] += std::ceil(kv.second * 1000.0 - 1e-9);
    }
    return r;
  }
  Resource& Add(const Resource& rr) { MilliCPU += rr.MilliCPU; Memory += rr.Memory; for (auto& kv : rr.ScalarResources) ScalarResources[kv.first] += kv.second; return *this; }
  Resource& SubUnchecked(const Resource& rr) { MilliCPU -= rr.MilliCPU; Memory -= rr.Memory; for (auto& kv : rr.ScalarResources) ScalarResources[kv.first] -= kv.second; return *this; }
  // Resource.LessEqual (resource_info.go:268-302): epsilons 10 m / 10 Mi / 10; scalars <= 10 are skipped; a nil map on the
  // right makes any larger scalar fail
  bool LessEqual(const Resource& rr) const {
    auto le = [](double l, double r, double diff) { return l < r || std::fabs(l - r) < diff; };
    if (!le(MilliCPU, rr.MilliCPU, 10.0)) return false;
    if (!le(Memory, rr.Memory, 10.0 * 1024 * 1024)) return false;
    for (auto& kv : ScalarResources) {
      if (kv.second <= 10.0) continue;
      if (rr.ScalarResources.empty()) return false;
      auto it = rr.ScalarResources.find(kv.first);
      if (!le(kv.second, it == rr.ScalarResources.end() ? 0.0 : it->second, 10.0)) return false;
    }
    return true;
  }
  void SetMaxResource(const Resource& rr) { MilliCPU = std::max(MilliCPU, rr.MilliCPU); Memory = std::max(Memory, rr.Memory);
    for (auto& kv : rr.ScalarResources) { auto& x = ScalarResources[kv.first]; x = std::max(x, kv.second); } }
};

enum TaskStatus { Pending = 1, Allocated = 2, Pipelined = 4, Binding = 8, Bound = 16, Running = 32, Releasing = 64,
                  Succeeded = 128, Failed = 256, Unknown = 512 };                     // api/types.go:20-54
inline bool AllocatedStatus(int s) { return s == Bound || s == Binding || s == Running || s == Allocated; }   // api/helpers.go:64-71

// v1.Affinity (k8s.io/api/core/v1/types.go).  A nil pointer is the Go nil; an empty list is an empty list.
struct NodeSelectorRequirement { std::string Key, Operator; std::vector<std::string> Values; };   // In NotIn Exists DoesNotExist Gt Lt
struct NodeSelectorTerm { std::vector<NodeSelectorRequirement> MatchExpressions, MatchFields; };
struct NodeSelector { std::vector<NodeSelectorTerm> NodeSelectorTerms; };
struct PreferredSchedulingTerm { int32_t Weight = 0; NodeSelectorTerm Preference; };
struct NodeAffinity {
  std::shared_ptr<NodeSelector> RequiredDuringSchedulingIgnoredDuringExecution;
  std::vector<PreferredSchedulingTerm> PreferredDuringSchedulingIgnoredDuringExecution;
};
struct LabelSelectorRequirement { std::string Key, Operator; std::vector<std::string> Values; };  // In NotIn Exists DoesNotExist
struct LabelSelector { std::map<std::string, std::string> MatchLabels; std::vector<LabelSelectorRequirement> MatchExpressions; };
struct PodAffinityTerm {
  std::shared_ptr<api::LabelSelector> LabelSelector;  // nil: labels.Nothing() (LabelSelectorAsSelector)
  std::vector<std::string> Namespaces;                // empty: the owning pod's namespace
  std::string TopologyKey;
};
struct WeightedPodAffinityTerm { int32_t Weight = 0; api::PodAffinityTerm PodAffinityTerm; };
struct PodAffinity {                                  // also v1.PodAntiAffinity
  std::vector<api::PodAffinityTerm> RequiredDuringSchedulingIgnoredDuringExecution;
  std::vector<WeightedPodAffinityTerm> PreferredDuringSchedulingIgnoredDuringExecution;
};
struct Affinity {
  std::shared_ptr<api::NodeAffinity> NodeAffinity;
  std::shared_ptr<api::PodAffinity> PodAffinity, PodAntiAffinity;
};

struct Pod {                                          // the v1.Pod fields the path reads (util/test_utils.go:66-93 BuildPod)
  std::string Namespace, Name, UID, NodeName, Phase = "Pending", GroupName;
  std::shared_ptr<api::Affinity> Affinity;            // Spec.Affinity
  ResourceList Requests;                              // one container
  std::vector<ResourceList> InitRequests;
  std::map<std::string, std::string> Labels, NodeSelector;
  struct Toleration { std::string Key, Operator, Value, Effect; };
  std::vector<Toleration> Tolerations;
  struct HostPort { std::string HostIP, Protocol; int Port; };
  std::vector<HostPort> HostPorts;
  int32_t Priority = 1;
  std::string PriorityClassName;                      // Spec.PriorityClassName (conformance.go:45-53)
  int64_t CreationTimestamp = 0;
  bool Deleting = false;
};

struct Node {                                         // v1.Node fields the path reads (util/test_utils.go:52-63 BuildNode)
  std::string Name;
  ResourceList Allocatable;
  std::map<std::string, std::string> Labels;
  struct Taint { std::string Key, Value, Effect; };
  std::vector<Taint> Taints;
  bool Unschedulable = false, NotReady = false, NetworkUnavailable = false, MemoryPressure = false, DiskPressure = false, PIDPressure = false;
};

struct TaskInfo {                                     // api/job_info.go:36-54
  std::string UID, Job, Name, Namespace, NodeName;
  Resource Resreq, InitResreq;
  int Status = Pending;
  int32_t Priority = 1;
  std::shared_ptr<Pod> pod;
  std::shared_ptr<TaskInfo> Clone() const { return std::make_shared<TaskInfo>(*this); }   // job_info.go:96-113 (the Pod is shared)
};

struct NodeInfo {                                     // api/node_info.go:28-47
  std::string Name;
  std::shared_ptr<Node> node;
  Resource Releasing, Idle, Used, Allocatable;
  std::map<std::string, std::shared_ptr<TaskInfo>> Tasks;
  // api/node_info.go:172-212.  The node keeps its own copy of the task, so a later status change of the caller's object
  // leaves the node's resources alone until UpdateTask / RemoveTask.
  void AddTask(const std::shared_ptr<TaskInfo>& task) {
    if (Tasks.count(task->Namespace + "/" + task->Name)) throw std::runtime_error("task already on node " + Name);
    switch (task->Status) {
      case Releasing_: Idle.SubUnchecked(task->Resreq); Releasing.Add(task->Resreq); break;
      case Pipelined: Releasing.SubUnchecked(task->Resreq); break;
      default: Idle.SubUnchecked(task->Resreq); break;
    }
    Used.Add(task->Resreq);
    task->NodeName = Name;
    Tasks[task->Namespace + "/" + task->Name] = task->Clone();
  }
  // api/node_info.go:214-245: gives back what the node's own copy holds, by that copy's status
  void RemoveTask(const TaskInfo& ti) {
    auto it = Tasks.find(ti.Namespace + "/" + ti.Name);
    if (it == Tasks.end()) throw std::runtime_error("failed to find task " + ti.Namespace + "/" + ti.Name + " on host " + Name);
    const TaskInfo& task = *it->second;
    switch (task.Status) {
      case Releasing_: Releasing.SubUnchecked(task.Resreq); Idle.Add(task.Resreq); break;
      case Pipelined: Releasing.Add(task.Resreq); break;
      default: Idle.Add(task.Resreq); break;
    }
    Used.SubUnchecked(task.Resreq);
    Tasks.erase(it);
  }
  // api/node_info.go:245-259
  void UpdateTask(const std::shared_ptr<TaskInfo>& ti) { RemoveTask(*ti); AddTask(ti); }
  static constexpr int Releasing_ = api::Releasing;
};

struct JobInfo {                                      // api/job_info.go:127-154
  std::string UID, Name, Namespace, Queue;
  int32_t Priority = 0, MinAvailable = 0;
  int64_t CreationTimestamp = 0;
  std::map<std::string, std::shared_ptr<TaskInfo>> Tasks;
  std::map<int, std::map<std::string, std::shared_ptr<TaskInfo>>> TaskStatusIndex;
  Resource Allocated;
  void AddTaskInfo(const std::shared_ptr<TaskInfo>& t) { Tasks[t->UID] = t; TaskStatusIndex[t->Status][t->UID] = t; if (AllocatedStatus(t->Status)) Allocated.Add(t->Resreq); }
  // job_info.go:247-264: the job's entry for the UID (found by UID, removed by ITS status) is replaced by `t` — which may be
  // another object for the same task, e.g. the clone of a node's copy that reclaim / preempt evict
  void UpdateTaskStatus(const std::shared_ptr<TaskInfo>& t, int status) {
    auto found = Tasks.find(t->UID);
    if (found != Tasks.end()) {                         // DeleteTaskInfo, job_info.go:279-295
      const std::shared_ptr<TaskInfo> old = found->second;
      if (AllocatedStatus(old->Status)) Allocated.SubUnchecked(old->Resreq);
      Tasks.erase(found);
      auto it = TaskStatusIndex.find(old->Status);
      if (it != TaskStatusIndex.end()) { it->second.erase(old->UID); if (it->second.empty()) TaskStatusIndex.erase(it); }
    }
    t->Status = status;
    AddTaskInfo(t);
  }
  int32_t ReadyTaskNum() const {                      // job_info.go:383-393
    int n = 0;
    for (auto& kv : TaskStatusIndex) if (AllocatedStatus(kv.first) || kv.first == Succeeded) n += (int)kv.second.size();
    return n;
  }
  bool Ready() const { return ReadyTaskNum() >= MinAvailable; }   // job_info.go:423-427
};

struct QueueInfo { std::string UID, Name; int32_t Weight = 1; int64_t CreationTimestamp = 0; };   // api/queue_info.go:74-81

}  // namespace api

// ------------------------------------------------------------------------------------------------ conf
namespace conf {
struct PluginOption {                                 // conf/scheduler_conf.go:33-56; -1 = nil *bool
  std::string Name;
  int EnabledJobOrder = -1, EnabledJobReady = -1, EnabledJobPipelined = -1, EnabledTaskOrder = -1, EnabledPreemptable = -1,
      EnabledReclaimable = -1, EnabledQueueOrder = -1, EnabledPredicate = -1, EnabledNodeOrder = -1;
  std::map<std::string, std::string> Arguments;
};
struct Tier { std::vector<PluginOption> Plugins; };
inline void ApplyPluginConfDefaults(PluginOption& o) {           // plugins/defaults.go:22-52: nil -> true
  for (int* p : {&o.EnabledJobOrder, &o.EnabledJobReady, &o.EnabledJobPipelined, &o.EnabledTaskOrder, &o.EnabledPreemptable,
                 &o.EnabledReclaimable, &o.EnabledQueueOrder, &o.EnabledPredicate, &o.EnabledNodeOrder}) if (*p < 0) *p = 1;
}
}  // namespace conf

// ----------------------------------------------------------------------------------------------- cache
namespace cache {
struct Binder { virtual ~Binder() = default; virtual void Bind(const api::TaskInfo& task, const std::string& hostname) = 0; };
struct FakeBinder : Binder {                          // util/test_utils.go:95-112
  std::map<std::string, std::string> Binds;
  void Bind(const api::TaskInfo& task, const std::string& hostname) override { Binds[task.Namespace + "/" + task.Name] = hostname; }
};
struct Evictor { virtual ~Evictor() = default; virtual void Evict(const api::Pod& pod) = 0; };   // cache/interface.go:68-72
struct FakeEvictor : Evictor {                        // util/test_utils.go:114-133
  std::vector<std::string> Evicts;                    // in call order
  void Evict(const api::Pod& pod) override { Evicts.push_back(pod.Namespace + "/" + pod.Name); }
};
struct PodGroup { std::string Namespace, Name, Queue; int32_t MinMember = 0; int32_t Priority = 0; int64_t CreationTimestamp = 0; };
struct ClusterInfo {                                  // api/cluster_info.go:22-26
  std::map<std::string, std::shared_ptr<api::JobInfo>> Jobs;
  std::map<std::string, std::shared_ptr<api::NodeInfo>> Nodes;
  std::map<std::string, std::shared_ptr<api::QueueInfo>> Queues;
};
struct SchedulerCache {                               // the literal cache of allocate_test.go:154-177
  std::map<std::string, std::shared_ptr<api::NodeInfo>> Nodes;
  std::map<std::string, std::shared_ptr<api::JobInfo>> Jobs;
  std::map<std::string, std::shared_ptr<api::QueueInfo>> Queues;
  std::shared_ptr<Binder> binder;
  std::shared_ptr<Evictor> evictor;
  // cache/cache.go:425-480.  The session shares this cache's objects (Snapshot does not deep-copy), so the status and node
  // updates of the reference's cache.Evict are the session's own (Session::Evict, Statement::Evict); what is left is the
  // call to the Evictor.
  void Evict(const api::TaskInfo& task, const std::string& /*reason*/) { if (evictor) evictor->Evict(*task.pod); }
  void AddNode(const api::Node& n) {
    auto ni = std::make_shared<api::NodeInfo>();
    ni->Name = n.Name; ni->node = std::make_shared<api::Node>(n);
    ni->Allocatable = api::Resource::New(n.Allocatable); ni->Idle = ni->Allocatable; ni->Idle.MaxTaskNum = ni->Allocatable.MaxTaskNum;
    Nodes[n.Name] = ni;
  }
  void AddQueue(const std::string& name, int32_t weight) { auto q = std::make_shared<api::QueueInfo>(); q->UID = q->Name = name; q->Weight = weight; Queues[name] = q; }
  std::shared_ptr<api::JobInfo> getOrCreateJob(const std::string& ns, const std::string& group) {
    const std::string id = ns + "/" + group;
    auto it = Jobs.find(id);
    if (it != Jobs.end()) return it->second;
    auto j = std::make_shared<api::JobInfo>(); j->UID = id; j->Namespace = ns; j->Name = group; Jobs[id] = j; return j;
  }
  void AddPodGroup(const PodGroup& pg) {
    auto j = getOrCreateJob(pg.Namespace, pg.Name);
    j->Queue = pg.Queue; j->MinAvailable = pg.MinMember; j->Priority = pg.Priority; j->CreationTimestamp = pg.CreationTimestamp;
    has_spec.insert(j->UID);
  }
  static int taskStatus(const api::Pod& p) {          // api/helpers.go:38-62
    if (p.Phase == "Running") return p.Deleting ? api::Releasing : api::Running;
    if (p.Phase == "Pending") { if (p.Deleting) return api::Releasing; return p.NodeName.empty() ? api::Pending : api::Bound; }
    if (p.Phase == "Succeeded") return api::Succeeded;
    if (p.Phase == "Failed") return api::Failed;
    return api::Unknown;
  }
  void AddPod(const api::Pod& pod) {
    auto t = std::make_shared<api::TaskInfo>();
    t->pod = std::make_shared<api::Pod>(pod);
    t->UID = pod.UID.empty() ? pod.Namespace + "-" + pod.Name : pod.UID;
    t->Name = pod.Name; t->Namespace = pod.Namespace; t->NodeName = pod.NodeName; t->Priority = pod.Priority;
    t->Resreq = api::Resource::New(pod.Requests);
    t->InitResreq = t->Resreq;
    for (auto& ir : pod.InitRequests) t->InitResreq.SetMaxResource(api::Resource::New(ir));   // api/pod_info.go:53-73
    t->Status = taskStatus(pod);
    auto j = getOrCreateJob(pod.Namespace, pod.GroupName);
    t->Job = j->UID;
    j->AddTaskInfo(t);
    // cache.addTask (cache/event_handlers.go): the job gets the task, then node.AddTask — which refuses a task that does not
    // fit into Idle (allocateIdleResource, node_info.go:161-167; a Pipelined task takes Releasing instead), so a node is never
    // over-committed in the snapshot
    if (!pod.NodeName.empty() && Nodes.count(pod.NodeName) && t->Status != api::Pending) {
      auto& n = *Nodes[pod.NodeName];
      if (t->Status == api::Pipelined || t->Resreq.LessEqual(n.Idle)) n.AddTask(t);
    }
  }
  ClusterInfo Snapshot() const {                      // cache/cache.go:627-683 (objects are shared, not deep-copied)
    ClusterInfo ci;
    ci.Nodes = Nodes; ci.Queues = Queues;
    for (auto& kv : Jobs) { if (!has_spec.count(kv.first)) continue; if (!Queues.count(kv.second->Queue)) continue; ci.Jobs[kv.first] = kv.second; }
    return ci;
  }
  std::set<std::string> has_spec;
};
}  // namespace cache

// ------------------------------------------------------------------------------------------- framework
namespace framework {

using Arguments = std::map<std::string, std::string>;                 // framework/arguments.go:26
class Session;

// Which built-in function a plugin registers.  A value of Foreign marks a callback the GPU path cannot honour.
enum class Builtin { PriorityTaskOrder, PriorityJobOrder, GangJobOrder, GangJobReady, GangJobPipelined, DrfJobOrder, DrfPreemptable,
                     ProportionQueueOrder, ProportionOverused, ProportionReclaimable, Predicates, NodeOrder, Foreign };

class Plugin {                                        // framework/interface.go:34-41
 public:
  virtual ~Plugin() = default;
  virtual std::string Name() const = 0;
  virtual void OnSessionOpen(Session* ssn) = 0;
  virtual void OnSessionClose(Session*) {}
};
class Action {                                        // framework/interface.go:20-32
 public:
  virtual ~Action() = default;
  virtual std::string Name() const = 0;
  virtual void Initialize() {}
  virtual void Execute(Session* ssn) = 0;
  virtual void UnInitialize() {}
};

using PluginBuilder = std::function<std::unique_ptr<Plugin>(const Arguments&)>;
inline std::map<std::string, PluginBuilder>& pluginBuilders() { static std::map<std::string, PluginBuilder> m; return m; }
inline void RegisterPluginBuilder(const std::string& name, PluginBuilder pb) { pluginBuilders()[name] = std::move(pb); }   // framework/plugins.go:30
inline void CleanupPluginBuilders() { pluginBuilders().clear(); }

class Session {                                       // framework/session.go:37-61
 public:
  std::string UID = "session";
  std::map<std::string, std::shared_ptr<api::JobInfo>> Jobs;
  std::map<std::string, std::shared_ptr<api::NodeInfo>> Nodes;
  std::map<std::string, std::shared_ptr<api::QueueInfo>> Queues;
  std::vector<conf::Tier> Tiers;
  cache::SchedulerCache* cache = nullptr;
  std::map<std::string, std::unique_ptr<Plugin>> plugins;
  std::map<std::string, std::vector<Builtin>> registered;              // plugin name -> what it registered
  std::map<std::string, Arguments> pluginArguments;

  // session_plugins.go:25-77 — the registration surface (source-compatible names)
  void AddJobOrderFn(const std::string& name, Builtin fn) { registered[name].push_back(fn); }
  void AddQueueOrderFn(const std::string& name, Builtin fn) { registered[name].push_back(fn); }
  void AddTaskOrderFn(const std::string& name, Builtin fn) { registered[name].push_back(fn); }
  void AddPreemptableFn(const std::string& name, Builtin fn) { registered[name].push_back(fn); }
  void AddReclaimableFn(const std::string& name, Builtin fn) { registered[name].push_back(fn); }
  void AddJobReadyFn(const std::string& name, Builtin fn) { registered[name].push_back(fn); }
  void AddJobPipelinedFn(const std::string& name, Builtin fn) { registered[name].push_back(fn); }
  void AddPredicateFn(const std::string& name, Builtin fn) { registered[name].push_back(fn); }
  void AddNodePrioritizers(const std::string& name, Builtin fn) { registered[name].push_back(fn); }
  void AddNodeOrderFn(const std::string& name, Builtin fn) { AddNodePrioritizers(name, fn); }   // alias (SURVEY: API-name drift)
  void AddOverusedFn(const std::string& name, Builtin fn) { registered[name].push_back(fn); }
  void AddJobValidFn(const std::string&, Builtin) {}                   // dead at this commit (session.go:89-108)

  // session_plugins.go:182-200 — JobReady = AND of enabled JobReadyFns; only gang registers one
  bool JobReady(const api::JobInfo& job) const {
    for (auto& tier : Tiers) for (auto& p : tier.Plugins) {
      if (p.EnabledJobReady != 1) continue;
      auto it = registered.find(p.Name);
      if (it == registered.end()) continue;
      for (Builtin b : it->second) if (b == Builtin::GangJobReady && !job.Ready()) return false;
    }
    return true;
  }
  // framework/session.go:235-288
  void Allocate(const std::shared_ptr<api::TaskInfo>& task, const std::string& hostname) {
    auto& job = Jobs.at(task->Job);
    job->UpdateTaskStatus(task, api::Allocated);
    Nodes.at(hostname)->AddTask(task);
    if (JobReady(*job)) {
      auto it = job->TaskStatusIndex.find(api::Allocated);
      if (it != job->TaskStatusIndex.end()) {
        std::vector<std::shared_ptr<api::TaskInfo>> ts;
        for (auto& kv : it->second) ts.push_back(kv.second);
        for (auto& t : ts) dispatch(t);
      }
    }
  }
  // framework/session.go:194-232
  void Pipeline(const std::shared_ptr<api::TaskInfo>& task, const std::string& hostname) {
    Jobs.at(task->Job)->UpdateTaskStatus(task, api::Pipelined);
    Nodes.at(hostname)->AddTask(task);
  }
  // framework/session.go:290-314
  void dispatch(const std::shared_ptr<api::TaskInfo>& task) {
    if (cache && cache->binder) cache->binder->Bind(*task, task->NodeName);
    Jobs.at(task->Job)->UpdateTaskStatus(task, api::Binding);
  }
  // framework/session.go:317-353.  Callers pass a clone of the node's task (reclaim.go:135-136): the node's own copy must
  // still hold the old status when UpdateTask takes it off the node.
  void Evict(const std::shared_ptr<api::TaskInfo>& reclaimee, const std::string& reason) {
    if (cache) cache->Evict(*reclaimee, reason);
    Jobs.at(reclaimee->Job)->UpdateTaskStatus(reclaimee, api::Releasing);
    auto node = Nodes.find(reclaimee->NodeName);
    if (node != Nodes.end()) node->second->UpdateTask(reclaimee);
  }
};

// framework/statement.go: evictions and pipelines applied to the session at once, sent to the cache by Commit or undone in
// reverse order by Discard.  ssn.Statement() (session.go:186-191) is `Statement stmt(ssn)` here.
class Statement {
 public:
  explicit Statement(Session* ssn) : ssn_(ssn) {}
  void Evict(const std::shared_ptr<api::TaskInfo>& reclaimee, const std::string& reason) {   // statement.go:37-69
    updateStatus(reclaimee, api::Releasing);
    auto node = ssn_->Nodes.find(reclaimee->NodeName);
    if (node != ssn_->Nodes.end()) node->second->UpdateTask(reclaimee);
    operations_.push_back({true, reclaimee, reason});
  }
  void Pipeline(const std::shared_ptr<api::TaskInfo>& task, const std::string& hostname) {  // statement.go:113-152
    updateStatus(task, api::Pipelined);
    ssn_->Nodes.at(hostname)->AddTask(task);
    operations_.push_back({false, task, hostname});
  }
  void Commit() {                                                                           // statement.go:210-221
    for (auto& op : operations_) if (op.evict && ssn_->cache) ssn_->cache->Evict(*op.task, op.arg);
  }
  void Discard() {                                                                          // statement.go:196-208
    for (auto it = operations_.rbegin(); it != operations_.rend(); ++it) {
      auto& task = it->task;
      if (it->evict) {                                  // unevict, statement.go:83-111
        updateStatus(task, api::Running);
        auto node = ssn_->Nodes.find(task->NodeName);
        if (node != ssn_->Nodes.end()) node->second->UpdateTask(task);
      } else {                                          // unpipeline, statement.go:157-194
        updateStatus(task, api::Pending);
        auto node = ssn_->Nodes.find(task->NodeName);
        if (node != ssn_->Nodes.end()) node->second->RemoveTask(*task);
      }
    }
  }

 private:
  struct operation { bool evict; std::shared_ptr<api::TaskInfo> task; std::string arg; };   // arg: reason / hostname
  void updateStatus(const std::shared_ptr<api::TaskInfo>& task, int status) {
    auto job = ssn_->Jobs.find(task->Job);
    if (job != ssn_->Jobs.end()) job->second->UpdateTaskStatus(task, status);
  }
  Session* ssn_;
  std::vector<operation> operations_;
};

// framework/framework.go:30-52
inline std::unique_ptr<Session> OpenSession(cache::SchedulerCache* cache, const std::vector<conf::Tier>& tiers) {
  static uint64_t sessions = 0;
  auto ssn = std::make_unique<Session>();
  ssn->UID = "session-" + std::to_string(++sessions);   // uuid.NewUUID() (session.go:65): what a cycle's result is cached under
  ssn->cache = cache;
  auto snap = cache->Snapshot();
  ssn->Jobs = snap.Jobs; ssn->Nodes = snap.Nodes; ssn->Queues = snap.Queues;
  ssn->Tiers = tiers;
  for (auto& tier : tiers) for (auto& po : tier.Plugins) {
    auto it = pluginBuilders().find(po.Name);
    if (it == pluginBuilders().end()) continue;        // "Failed to get plugin" is only logged in the reference
    auto pl = it->second(po.Arguments);
    ssn->pluginArguments[pl->Name()] = po.Arguments;
    ssn->plugins[pl->Name()] = std::move(pl);
  }
  for (auto& kv : ssn->plugins) kv.second->OnSessionOpen(ssn.get());
  return ssn;
}
inline void CloseSession(Session* ssn) { for (auto& kv : ssn->plugins) kv.second->OnSessionClose(ssn); }

}  // namespace framework

// --------------------------------------------------------------------------------------------- plugins
namespace plugins {
using framework::Arguments; using framework::Builtin; using framework::Plugin; using framework::Session;
#define KB_PLUGIN(cls, pname, body) struct cls : Plugin { Arguments args; explicit cls(const Arguments& a) : args(a) {} \
  std::string Name() const override { return pname; } void OnSessionOpen(Session* ssn) override body }
KB_PLUGIN(priorityPlugin, "priority", { ssn->AddTaskOrderFn(Name(), Builtin::PriorityTaskOrder); ssn->AddJobOrderFn(Name(), Builtin::PriorityJobOrder); });
KB_PLUGIN(gangPlugin, "gang", { ssn->AddJobOrderFn(Name(), Builtin::GangJobOrder); ssn->AddJobReadyFn(Name(), Builtin::GangJobReady); ssn->AddJobPipelinedFn(Name(), Builtin::GangJobPipelined); });
KB_PLUGIN(drfPlugin, "drf", { ssn->AddPreemptableFn(Name(), Builtin::DrfPreemptable); ssn->AddJobOrderFn(Name(), Builtin::DrfJobOrder); });
KB_PLUGIN(proportionPlugin, "proportion", { ssn->AddQueueOrderFn(Name(), Builtin::ProportionQueueOrder); ssn->AddReclaimableFn(Name(), Builtin::ProportionReclaimable); ssn->AddOverusedFn(Name(), Builtin::ProportionOverused); });
KB_PLUGIN(predicatesPlugin, "predicates", { ssn->AddPredicateFn(Name(), Builtin::Predicates); });
KB_PLUGIN(nodeOrderPlugin, "nodeorder", { ssn->AddNodePrioritizers(Name(), Builtin::NodeOrder); });
KB_PLUGIN(conformancePlugin, "conformance", { (void)ssn; });
#undef KB_PLUGIN
inline void RegisterBuiltins() {                       // plugins/factory.go:31-42
  using framework::RegisterPluginBuilder;
  RegisterPluginBuilder("priority", [](const Arguments& a) { return std::make_unique<priorityPlugin>(a); });
  RegisterPluginBuilder("gang", [](const Arguments& a) { return std::make_unique<gangPlugin>(a); });
  RegisterPluginBuilder("drf", [](const Arguments& a) { return std::make_unique<drfPlugin>(a); });
  RegisterPluginBuilder("proportion", [](const Arguments& a) { return std::make_unique<proportionPlugin>(a); });
  RegisterPluginBuilder("predicates", [](const Arguments& a) { return std::make_unique<predicatesPlugin>(a); });
  RegisterPluginBuilder("nodeorder", [](const Arguments& a) { return std::make_unique<nodeOrderPlugin>(a); });
  RegisterPluginBuilder("conformance", [](const Arguments& a) { return std::make_unique<conformancePlugin>(a); });
}
}  // namespace plugins

// ------------------------------------------------------------------------------------- actions/allocate
namespace actions { namespace allocate {

// Flattened session: the SoA arrays of kb_snapshot plus the back-references needed to replay decisions.
struct Flat {
  uint32_t R = 2, W = 1, N = 0, T = 0, J = 0, Q = 0;
  std::vector<std::string> dims, nodeNames, jobIDs;
  std::vector<std::shared_ptr<api::TaskInfo>> tasks;
  std::vector<double> node_idle, node_releasing, node_used, node_allocatable, task_initreq, task_resreq, job_alloc0;
  std::vector<uint32_t> node_alloc_present, node_flags, task_res_present, task_n_aff, task_flags, task_uid_rank, job_task_off, job_alloc0_present, job_queue;
  std::vector<int64_t> node_alloc_cpu, node_alloc_mem, node_nz_cpu, node_nz_mem, task_nz_cpu, task_nz_mem, task_ctime, job_ctime, queue_ctime;
  std::vector<int32_t> node_pods, node_max_pods, task_prio, job_min_avail, job_ready0, job_prio, queue_weight;
  std::vector<uint64_t> node_labels, node_taints, node_ports, task_sel_req, task_aff, task_tol, task_port_own, task_port_conflict;
  std::vector<uint32_t> task_n_pref;                  // [T]
  std::vector<uint64_t> task_pref;                    // [KB_MAX_PREF_TERMS][W][T]
  std::vector<int32_t> task_pref_w;                   // [KB_MAX_PREF_TERMS][T]
  uint32_t snap_flags = 0;                            // KB_SNAPSHOT_*
  // kb_pod_affinity (FlattenPodAffinity); `on` is false when no pod of the session carries inter-pod terms
  struct PodAff {
    bool on = false;
    uint32_t n_keysets = 0, n_groups = 0, n_kinds = 0;
    int32_t first_unbound = -1;
    std::vector<int32_t> node_domain, group_count0, group_total0, task_need, task_kind, node_kind_count0, weight_kind, weight_keyset;
    std::vector<uint32_t> keyset_domains, group_keyset, task_weight_off, task_xgroup_off, task_xgroup;   // xgroup: empty when <= 64 groups
    std::vector<uint64_t> task_forbid, task_contrib;
    std::vector<uint8_t> kind_unbound;
    std::vector<int64_t> weight_value;
    std::map<const api::Pod*, std::vector<uint32_t>> member_groups;   // listed pods that are members: their groups, ascending
    kb_pod_affinity c{};                              // filled by SnapshotOf over the vectors above
  } pa;
};

inline void resourceVec(const api::Resource& r, const std::vector<std::string>& dims, double* out, size_t stride, uint32_t* present) {
  out[0] = r.MilliCPU; out[stride] = r.Memory;
  uint32_t p = 0;
  for (auto& kv : r.ScalarResources) { size_t k = std::find(dims.begin(), dims.end(), kv.first) - dims.begin(); out[k * stride] = kv.second; p |= 1u << k; }
  if (present) *present = p;
}

// "kbgpu: unsupported session: ..." — what the Go shim returns as *ErrUnsupported
inline std::runtime_error Unsupported(const std::string& why) { return std::runtime_error("kbgpu: unsupported session: " + why); }

// strconv.ParseInt(s, 10, 64)
inline bool parseInt64(const std::string& s, int64_t* out) {
  size_t i = (!s.empty() && (s[0] == '+' || s[0] == '-')) ? 1 : 0;
  if (i == s.size()) return false;
  for (size_t k = i; k < s.size(); ++k) if (s[k] < '0' || s[k] > '9') return false;
  errno = 0;
  char* end = nullptr;
  long long v = std::strtoll(s.c_str(), &end, 10);
  if (errno == ERANGE) return false;
  *out = v;
  return true;
}

// labels.Requirement.Matches of a requirement labels.NewRequirement accepts; a requirement it refuses matches nothing (the vendored
// callers treat the error as "no match": MatchNodeSelectorTerms, NodeSelectorRequirementsAsSelector)
inline bool labelRequirementHolds(const std::map<std::string, std::string>& labels, const std::string& key, const std::string& op,
                                  const std::vector<std::string>& values) {
  auto it = labels.find(key);
  const bool has = it != labels.end();
  auto in = [&] { return has && std::find(values.begin(), values.end(), it->second) != values.end(); };
  if (op == "In") return !values.empty() && in();
  if (op == "NotIn") return !values.empty() && !in();
  if (op == "Exists") return values.empty() && has;
  if (op == "DoesNotExist") return values.empty() && !has;
  if (op == "Gt" || op == "Lt") {                     // one integer value; a label that does not parse fails the match
    int64_t rv, lv;
    if (values.size() != 1 || !parseInt64(values[0], &rv) || !has || !parseInt64(it->second, &lv)) return false;
    return op == "Gt" ? lv > rv : lv < rv;
  }
  return false;
}

// One node-selector requirement evaluated ONCE per node (flatten.go reqAtom / atomTable): a nodeSelector pair (as In), a required or
// preferred node-affinity MatchExpression, or a MatchFields requirement.  Identical requirements written identically share the atom.
struct AtomTable {
  struct Req { bool field; std::string key, op; std::vector<std::string> values; };
  std::map<std::tuple<bool, std::string, std::string, std::vector<std::string>>, uint32_t> ids;
  std::vector<Req> reqs;
  uint32_t of(const api::NodeSelectorRequirement& r, bool field) {
    auto k = std::make_tuple(field, r.Key, r.Operator, r.Values);
    auto it = ids.find(k);
    if (it != ids.end()) return it->second;
    uint32_t id = (uint32_t)reqs.size();
    ids.emplace(k, id);
    reqs.push_back({field, r.Key, r.Operator, r.Values});
    return id;
  }
  // an atom no node satisfies: a required term without expressions, or a preferred term without expressions
  // (NodeSelectorRequirementsAsSelector of an empty list is labels.Nothing(), helpers.go:205-208)
  uint32_t never() { return of({"\x01never", "In", {"\x01"}}, false); }
  bool holds(uint32_t a, const api::Node& node) const {
    const Req& r = reqs[a];
    if (!r.field) return labelRequirementHolds(node.Labels, r.key, r.op, r.values);
    // NodeSelectorRequirementsAsFieldSelector (helpers.go:239-267): In / NotIn with one value, against fields.Set{"metadata.name": ...}
    if ((r.op != "In" && r.op != "NotIn") || r.values.size() != 1) return false;
    const std::string v = r.key == "metadata.name" ? node.Name : std::string();
    return r.op == "In" ? v == r.values[0] : v != r.values[0];
  }
};

inline void FlattenPodAffinity(const framework::Session& ssn, Flat& f);

// What the Go shim's Flatten(ssn) does (INTEGRATION.md §"What Flatten must compute"); mirrors builder.py::flatten.
inline Flat Flatten(const framework::Session& ssn) {
  Flat f;
  std::set<std::string> sc;
  for (auto& kv : ssn.Nodes) for (auto& s : kv.second->Allocatable.ScalarResources) sc.insert(s.first);
  for (auto& jk : ssn.Jobs) for (auto& tk : jk.second->Tasks) { for (auto& s : tk.second->Resreq.ScalarResources) sc.insert(s.first); for (auto& s : tk.second->InitResreq.ScalarResources) sc.insert(s.first); }
  f.dims = {"cpu", "memory"}; for (auto& s : sc) f.dims.push_back(s);
  f.R = (uint32_t)f.dims.size();
  if (f.R > KB_MAX_R) throw Unsupported(std::to_string(f.R) + " resource dimensions > KB_MAX_R (" + std::to_string(KB_MAX_R) + ")");
  std::vector<std::shared_ptr<api::NodeInfo>> nodes; for (auto& kv : ssn.Nodes) nodes.push_back(kv.second);       // std::map: ascending Name
  std::vector<std::shared_ptr<api::QueueInfo>> queues; for (auto& kv : ssn.Queues) queues.push_back(kv.second);
  std::vector<std::shared_ptr<api::JobInfo>> jobs; for (auto& kv : ssn.Jobs) jobs.push_back(kv.second);          // ascending JobID
  for (auto& j : jobs) f.jobIDs.push_back(j->UID);
  std::map<std::string, uint32_t> qidx; for (uint32_t i = 0; i < queues.size(); ++i) qidx[queues[i]->UID] = i;
  f.N = (uint32_t)nodes.size(); f.J = (uint32_t)jobs.size(); f.Q = (uint32_t)queues.size();
  // pending tasks grouped by job; UID ranks
  std::vector<std::string> uids;
  f.job_task_off.assign(f.J + 1, 0);
  for (uint32_t j = 0; j < f.J; ++j) {
    auto it = jobs[j]->TaskStatusIndex.find(api::Pending);
    if (it != jobs[j]->TaskStatusIndex.end()) for (auto& kv : it->second) { f.tasks.push_back(kv.second); uids.push_back(kv.second->UID); }
    f.job_task_off[j + 1] = (uint32_t)f.tasks.size();
  }
  f.T = (uint32_t)f.tasks.size();
  std::sort(uids.begin(), uids.end());
  // atoms: selector requirements, NoSchedule/NoExecute taints, host ports.  Per task in task order: the nodeSelector pairs (as In,
  // ascending key), the required node-affinity terms, the preferred ones (flatten.go, builder.py::flatten)
  AtomTable atoms;
  struct TaskTerms { std::vector<uint32_t> sel; std::vector<std::vector<uint32_t>> aff, pref; std::vector<int32_t> prefW; };
  std::vector<TaskTerms> terms(f.T);
  for (uint32_t t = 0; t < f.T; ++t) {
    const api::TaskInfo& ti = *f.tasks[t];
    const api::Pod& p = *ti.pod;
    for (auto& kv : p.NodeSelector) terms[t].sel.push_back(atoms.of({kv.first, "In", {kv.second}}, false));   // labels.SelectorFromSet
    if (!p.Affinity || !p.Affinity->NodeAffinity) continue;
    const api::NodeAffinity& na = *p.Affinity->NodeAffinity;
    if (na.RequiredDuringSchedulingIgnoredDuringExecution) {                      // predicates.go:944-968
      for (auto& term : na.RequiredDuringSchedulingIgnoredDuringExecution->NodeSelectorTerms) {
        if (term.MatchExpressions.empty() && term.MatchFields.empty()) continue;   // matches nothing (MatchNodeSelectorTerms)
        std::vector<uint32_t> as;
        for (auto& e : term.MatchExpressions) as.push_back(atoms.of(e, false));
        for (auto& e : term.MatchFields) as.push_back(atoms.of(e, true));
        terms[t].aff.push_back(as);
      }
      if (terms[t].aff.empty()) terms[t].aff.push_back({atoms.never()});
      if (terms[t].aff.size() > KB_MAX_AFF_TERMS)
        throw Unsupported("pod " + ti.Namespace + "/" + ti.Name + " has " + std::to_string(terms[t].aff.size()) + " required node-affinity terms > KB_MAX_AFF_TERMS");
    }
    for (auto& pt : na.PreferredDuringSchedulingIgnoredDuringExecution) {         // node_affinity.go:34-77
      if (pt.Weight == 0) continue;
      std::vector<uint32_t> as;
      for (auto& e : pt.Preference.MatchExpressions) as.push_back(atoms.of(e, false));   // MatchFields are ignored by the priority
      if (as.empty()) as.push_back(atoms.never());
      terms[t].pref.push_back(as);
      terms[t].prefW.push_back(pt.Weight);
    }
    if (terms[t].pref.size() > KB_MAX_PREF_TERMS)
      throw Unsupported("pod " + ti.Namespace + "/" + ti.Name + " has " + std::to_string(terms[t].pref.size()) + " preferred node-affinity terms > KB_MAX_PREF_TERMS");
  }
  std::map<std::tuple<std::string, std::string, std::string>, uint32_t> taintAtoms;
  std::map<std::tuple<std::string, std::string, int>, uint32_t> portAtoms;
  auto san = [](const api::Pod::HostPort& h) { return std::make_tuple(h.HostIP.empty() ? std::string("0.0.0.0") : h.HostIP, h.Protocol.empty() ? std::string("TCP") : h.Protocol, h.Port); };
  for (auto& n : nodes) for (auto& t : n->node->Taints) if (t.Effect == "NoSchedule" || t.Effect == "NoExecute") taintAtoms.emplace(std::make_tuple(t.Key, t.Value, t.Effect), (uint32_t)taintAtoms.size());
  for (auto& jk : ssn.Jobs) for (auto& tk : jk.second->Tasks) for (auto& h : tk.second->pod->HostPorts) if (h.Port > 0) portAtoms.emplace(san(h), (uint32_t)portAtoms.size());
  size_t need = std::max({atoms.reqs.size(), taintAtoms.size(), portAtoms.size(), (size_t)1});
  f.W = (uint32_t)((need + 63) / 64);
  if (f.W > KB_MAX_W) throw Unsupported(std::to_string(need) + " label / taint / port atoms > 64 x KB_MAX_W (" + std::to_string(KB_MAX_W) + ")");
  if (f.R > kb::KB_NARROW_R && f.W > kb::KB_NARROW_W)
    throw Unsupported(std::to_string(f.R) + " resource dimensions > KB_NARROW_R (" + std::to_string(kb::KB_NARROW_R) + ") with " + std::to_string(need) +
                      " atoms > 64 x KB_NARROW_W (" + std::to_string(kb::KB_NARROW_W) + ")");
  const uint32_t R = f.R, W = f.W, N = f.N, T = f.T, J = f.J, Q = f.Q;
  auto setbit = [](std::vector<uint64_t>& a, size_t stride, size_t i, uint32_t atom) { a[(atom / 64) * stride + i] |= 1ull << (atom % 64); };
  // nodes
  f.node_idle.assign((size_t)R * N, 0); f.node_releasing = f.node_used = f.node_allocatable = f.node_idle;
  f.node_alloc_present.assign(N, 0); f.node_flags.assign(N, 0); f.node_alloc_cpu.assign(N, 0); f.node_alloc_mem = f.node_nz_cpu = f.node_nz_mem = f.node_alloc_cpu;
  f.node_pods.assign(N, 0); f.node_max_pods.assign(N, 0);
  f.node_labels.assign((size_t)W * std::max(1u, N), 0); f.node_taints = f.node_ports = f.node_labels;
  for (uint32_t i = 0; i < N; ++i) {
    auto& n = *nodes[i];
    f.nodeNames.push_back(n.Name);
    resourceVec(n.Idle, f.dims, &f.node_idle[i], N, nullptr); resourceVec(n.Releasing, f.dims, &f.node_releasing[i], N, nullptr);
    resourceVec(n.Used, f.dims, &f.node_used[i], N, nullptr); resourceVec(n.Allocatable, f.dims, &f.node_allocatable[i], N, &f.node_alloc_present[i]);
    f.node_alloc_cpu[i] = (int64_t)n.Allocatable.MilliCPU; f.node_alloc_mem[i] = (int64_t)n.Allocatable.Memory;
    f.node_max_pods[i] = n.Allocatable.MaxTaskNum; f.node_pods[i] = (int32_t)n.Tasks.size();
    uint32_t fl = 0;
    fl |= n.node->NotReady ? KB_NODE_NOT_READY : 0u;
    fl |= n.node->NetworkUnavailable ? KB_NODE_NET_UNAVAILABLE : 0u;
    fl |= n.node->Unschedulable ? KB_NODE_UNSCHEDULABLE : 0u;
    fl |= n.node->MemoryPressure ? KB_NODE_MEM_PRESSURE : 0u;
    fl |= n.node->DiskPressure ? KB_NODE_DISK_PRESSURE : 0u;
    fl |= n.node->PIDPressure ? KB_NODE_PID_PRESSURE : 0u;
    f.node_flags[i] = fl;
    for (auto& kv : n.Tasks) {                         // nonzero requests + used ports of every task on the node
      auto& p = *kv.second->pod;
      f.node_nz_cpu[i] += p.Requests.count("cpu") ? (int64_t)std::ceil(p.Requests.at("cpu") * 1000.0 - 1e-9) : 100;           // non_zero.go:36
      f.node_nz_mem[i] += p.Requests.count("memory") ? (int64_t)p.Requests.at("memory") : 200ll * 1024 * 1024;             // non_zero.go:38
      for (auto& h : p.HostPorts) if (h.Port > 0) setbit(f.node_ports, N, i, portAtoms.at(san(h)));
    }
    for (uint32_t a = 0; a < atoms.reqs.size(); ++a) if (atoms.holds(a, *n.node)) setbit(f.node_labels, N, i, a);
    for (auto& t : n.node->Taints) { auto it = taintAtoms.find(std::make_tuple(t.Key, t.Value, t.Effect)); if (it != taintAtoms.end()) setbit(f.node_taints, N, i, it->second); }
  }
  // tasks
  f.task_initreq.assign((size_t)R * std::max(1u, T), 0); f.task_resreq = f.task_initreq;
  f.task_res_present.assign(std::max(1u, T), 0); f.task_n_aff = f.task_flags = f.task_uid_rank = f.task_res_present;
  f.task_nz_cpu.assign(std::max(1u, T), 0); f.task_nz_mem = f.task_ctime = f.task_nz_cpu; f.task_prio.assign(std::max(1u, T), 0);
  f.task_sel_req.assign((size_t)W * std::max(1u, T), 0); f.task_tol = f.task_port_own = f.task_port_conflict = f.task_sel_req;
  f.task_aff.assign((size_t)KB_MAX_AFF_TERMS * W * std::max(1u, T), 0);
  f.task_n_pref.assign(std::max(1u, T), 0); f.task_pref.assign((size_t)KB_MAX_PREF_TERMS * W * std::max(1u, T), 0);
  f.task_pref_w.assign((size_t)KB_MAX_PREF_TERMS * std::max(1u, T), 0);
  for (uint32_t t = 0; t < T; ++t) {
    auto& ti = *f.tasks[t]; auto& p = *ti.pod;
    resourceVec(ti.Resreq, f.dims, &f.task_resreq[t], T, &f.task_res_present[t]); resourceVec(ti.InitResreq, f.dims, &f.task_initreq[t], T, nullptr);
    f.task_nz_cpu[t] = p.Requests.count("cpu") ? (int64_t)std::ceil(p.Requests.at("cpu") * 1000.0 - 1e-9) : 100;
    f.task_nz_mem[t] = p.Requests.count("memory") ? (int64_t)p.Requests.at("memory") : 200ll * 1024 * 1024;
    for (uint32_t a : terms[t].sel) setbit(f.task_sel_req, T, t, a);
    f.task_n_aff[t] = (uint32_t)terms[t].aff.size();
    for (size_t k = 0; k < terms[t].aff.size(); ++k) for (uint32_t a : terms[t].aff[k]) f.task_aff[(k * W + a / 64) * T + t] |= 1ull << (a % 64);
    f.task_n_pref[t] = (uint32_t)terms[t].pref.size();
    for (size_t k = 0; k < terms[t].pref.size(); ++k) {
      f.task_pref_w[k * T + t] = terms[t].prefW[k];
      for (uint32_t a : terms[t].pref[k]) f.task_pref[(k * W + a / 64) * T + t] |= 1ull << (a % 64);
    }
    if (!terms[t].pref.empty()) f.task_flags[t] |= KB_TASK_HAS_PREFERRED_NODE_AFFINITY;
    for (auto& ta : taintAtoms) for (auto& tol : p.Tolerations) {                // Toleration.ToleratesTaint, toleration.go:37-56
      if (!tol.Effect.empty() && tol.Effect != std::get<2>(ta.first)) continue;
      if (!tol.Key.empty() && tol.Key != std::get<0>(ta.first)) continue;
      bool ok = tol.Operator == "Exists" || ((tol.Operator.empty() || tol.Operator == "Equal") && tol.Value == std::get<1>(ta.first));
      if (ok) setbit(f.task_tol, T, t, ta.second);
    }
    for (auto& h : p.HostPorts) { if (h.Port <= 0) continue; auto me = san(h); setbit(f.task_port_own, T, t, portAtoms.at(me));
      for (auto& pa : portAtoms) {                                                // HostPortInfo.CheckConflict, host_ports.go:96-125
        if (std::get<1>(pa.first) != std::get<1>(me) || std::get<2>(pa.first) != std::get<2>(me)) continue;
        if (std::get<0>(pa.first) == std::get<0>(me) || std::get<0>(pa.first) == "0.0.0.0" || std::get<0>(me) == "0.0.0.0") setbit(f.task_port_conflict, T, t, pa.second);
      } }
    if (p.Requests.empty()) f.task_flags[t] |= KB_TASK_BEST_EFFORT_QOS;
    f.task_prio[t] = ti.Priority; f.task_ctime[t] = p.CreationTimestamp;
    f.task_uid_rank[t] = (uint32_t)(std::lower_bound(uids.begin(), uids.end(), ti.UID) - uids.begin());
  }
  // jobs / queues
  f.job_min_avail.assign(std::max(1u, J), 0); f.job_ready0 = f.job_prio = f.job_min_avail; f.job_alloc0.assign((size_t)R * std::max(1u, J), 0);
  f.job_alloc0_present.assign(std::max(1u, J), 0); f.job_queue = f.job_alloc0_present; f.job_ctime.assign(std::max(1u, J), 0);
  for (uint32_t j = 0; j < J; ++j) {
    auto& job = *jobs[j];
    f.job_min_avail[j] = job.MinAvailable; f.job_ready0[j] = job.ReadyTaskNum(); f.job_prio[j] = job.Priority; f.job_ctime[j] = job.CreationTimestamp;
    f.job_queue[j] = qidx.at(job.Queue);
    resourceVec(job.Allocated, f.dims, &f.job_alloc0[j], J, &f.job_alloc0_present[j]);
  }
  f.queue_weight.assign(std::max(1u, Q), 0); f.queue_ctime.assign(std::max(1u, Q), 0);
  for (uint32_t q = 0; q < Q; ++q) { f.queue_weight[q] = queues[q]->Weight; f.queue_ctime[q] = queues[q]->CreationTimestamp; }
  FlattenPodAffinity(ssn, f);
  return f;
}

// ---- inter-pod (anti)affinity: the twin of go/kbgpu/podaffinity.go::flattenPodAffinity (builder.py::flatten_pod_affinity) ----

// What a term selects: GetNamespacesFromPodAffinityTerm + LabelSelectorAsSelector (topologies.go:25-49), with a canonical key:
// the namespaces, then the requirements ascending (a MatchLabels pair is the requirement key In (value))
struct TermProps {
  std::set<std::string> ns;
  bool nothing = false;                               // nil selector: labels.Nothing()
  std::vector<std::tuple<std::string, std::string, std::vector<std::string>>> reqs;   // (key, op, values ascending)
  std::string key;
  bool matches(const api::Pod& pod) const {           // PodMatchesTermsNamespaceAndSelector (topologies.go:38-49)
    if (!ns.count(pod.Namespace) || nothing) return false;
    for (auto& r : reqs) if (!labelRequirementHolds(pod.Labels, std::get<0>(r), std::get<1>(r), std::get<2>(r))) return false;
    return true;
  }
};

inline TermProps propsOf(const api::Pod& owner, const api::PodAffinityTerm& term) {
  TermProps p;
  for (auto& n : term.Namespaces) p.ns.insert(n);
  if (p.ns.empty()) p.ns.insert(owner.Namespace);
  for (auto& n : p.ns) p.key += n + ",";
  if (!term.LabelSelector) { p.nothing = true; p.key += "|nil"; return p; }
  for (auto& kv : term.LabelSelector->MatchLabels) p.reqs.emplace_back(kv.first, "In", std::vector<std::string>{kv.second});
  for (auto& e : term.LabelSelector->MatchExpressions) {     // labels.NewRequirement refuses what LabelSelectorAsSelector then returns
    const bool valued = e.Operator == "In" || e.Operator == "NotIn";
    if (!valued && e.Operator != "Exists" && e.Operator != "DoesNotExist")
      throw Unsupported("invalid label selector in a pod (anti)affinity term: \"" + e.Operator + "\" is not a valid pod selector operator");
    if (valued == e.Values.empty())
      throw Unsupported("invalid label selector in a pod (anti)affinity term: operator " + e.Operator + (valued ? " needs values" : " takes no values"));
    std::vector<std::string> v(e.Values);
    std::sort(v.begin(), v.end());
    v.erase(std::unique(v.begin(), v.end()), v.end());
    p.reqs.emplace_back(e.Key, e.Operator, v);
  }
  std::sort(p.reqs.begin(), p.reqs.end());
  p.key += "|sel";
  for (auto& r : p.reqs) {
    p.key += "|" + std::get<0>(r) + " " + std::get<1>(r);
    for (auto& v : std::get<2>(r)) p.key += " " + v;
  }
  return p;
}

inline const std::vector<api::PodAffinityTerm>& requiredTerms(const api::Pod& pod, bool anti) {
  static const std::vector<api::PodAffinityTerm> none;
  if (!pod.Affinity) return none;
  const auto& a = anti ? pod.Affinity->PodAntiAffinity : pod.Affinity->PodAffinity;
  return a ? a->RequiredDuringSchedulingIgnoredDuringExecution : none;
}
inline const std::vector<api::WeightedPodAffinityTerm>& preferredTerms(const api::Pod& pod, bool anti) {
  static const std::vector<api::WeightedPodAffinityTerm> none;
  if (!pod.Affinity) return none;
  const auto& a = anti ? pod.Affinity->PodAntiAffinity : pod.Affinity->PodAffinity;
  return a ? a->PreferredDuringSchedulingIgnoredDuringExecution : none;
}
inline bool hasPodAffinity(const api::Pod& pod) { return pod.Affinity && (pod.Affinity->PodAffinity || pod.Affinity->PodAntiAffinity); }

// pods with the same namespace, labels and (anti)affinity spec are interchangeable for every match below
inline std::string podType(const api::Pod& pod) {
  std::string s = pod.Namespace + '\x01';
  for (auto& kv : pod.Labels) s += kv.first + "=" + kv.second + ",";
  auto term = [&](const api::PodAffinityTerm& t) {
    s += "{" + t.TopologyKey + "|";
    for (auto& n : t.Namespaces) s += n + ",";
    if (!t.LabelSelector) { s += "|nil}"; return; }
    s += "|";
    for (auto& kv : t.LabelSelector->MatchLabels) s += kv.first + "=" + kv.second + ",";
    for (auto& e : t.LabelSelector->MatchExpressions) { s += e.Key + " " + e.Operator; for (auto& v : e.Values) s += " " + v; s += ","; }
    s += "}";
  };
  for (const auto* a : {pod.Affinity ? pod.Affinity->PodAffinity.get() : nullptr, pod.Affinity ? pod.Affinity->PodAntiAffinity.get() : nullptr}) {
    s += '\x01';
    if (!a) { s += "nil"; continue; }
    for (auto& t : a->RequiredDuringSchedulingIgnoredDuringExecution) term(t);
    s += "/";
    for (auto& w : a->PreferredDuringSchedulingIgnoredDuringExecution) { s += std::to_string(w.Weight); term(w.PodAffinityTerm); }
  }
  return s;
}

// Fills f.pa (f.pa.on stays false when no pod carries inter-pod terms), KB_TASK_HAS_POD_AFFINITY / KB_TASK_AFF_SELF_MATCH and
// KB_SNAPSHOT_PLACED_POD_AFFINITY / KB_SNAPSHOT_LISTED_POD_WITHOUT_NODE.  Throws Unsupported where flattenPodAffinity returns
// *ErrUnsupported.
inline void FlattenPodAffinity(const framework::Session& ssn, Flat& f) {
  const uint32_t N = f.N, T = f.T;
  std::map<std::string, uint32_t> nidx;
  for (uint32_t i = 0; i < N; ++i) nidx[f.nodeNames[i]] = i;
  struct Placed { const api::Pod* pod; uint32_t node; bool unbound; };
  // util.PodLister (plugins/util/util.go:37-85): AllocatedStatus tasks of the session's jobs, located by TaskInfo.NodeName
  std::vector<Placed> listed;
  bool any = false;
  for (auto& id : f.jobIDs) {
    for (auto& st : ssn.Jobs.at(id)->TaskStatusIndex) {
      if (!api::AllocatedStatus(st.first)) continue;
      for (auto& kv : st.second) {
        const api::TaskInfo& t = *kv.second;
        auto n = nidx.find(t.NodeName);
        if (n == nidx.end()) { f.snap_flags |= KB_SNAPSHOT_LISTED_POD_WITHOUT_NODE; continue; }   // GetNodeInfo fails (kbgpu.h)
        listed.push_back({t.pod.get(), n->second, t.pod->NodeName.empty()});
        if (hasPodAffinity(*t.pod)) { any = true; f.snap_flags |= KB_SNAPSHOT_PLACED_POD_AFFINITY; }
      }
    }
  }
  // NodeInfo.Tasks of every node, whatever the status: what nodeInfo.Pods() hands the priority
  std::vector<Placed> inTasks;
  int32_t firstUnbound = -1;
  for (uint32_t n = 0; n < N; ++n) {
    for (auto& kv : ssn.Nodes.at(f.nodeNames[n])->Tasks) {
      const api::Pod* pod = kv.second->pod.get();
      const bool unbound = pod->NodeName.empty();
      inTasks.push_back({pod, n, unbound});
      if (unbound && firstUnbound < 0) firstUnbound = (int32_t)n;
      if (hasPodAffinity(*pod)) { any = true; f.snap_flags |= KB_SNAPSHOT_PLACED_POD_AFFINITY; }
    }
  }
  for (auto& t : f.tasks) if (hasPodAffinity(*t->pod)) any = true;
  if (!any) return;
  Flat::PodAff& pa = f.pa;
  pa.on = true;
  pa.first_unbound = firstUnbound;

  // ---- pod types ----
  std::map<std::string, int> typeID;
  std::vector<const api::Pod*> reps;
  auto typeOf = [&](const api::Pod* pod) {
    auto ins = typeID.emplace(podType(*pod), (int)reps.size());
    if (ins.second) reps.push_back(pod);
    return ins.first->second;
  };
  std::vector<int> ptype(T), ltype, ttype;
  std::set<int> pendSet;
  for (uint32_t t = 0; t < T; ++t) { ptype[t] = typeOf(f.tasks[t]->pod.get()); pendSet.insert(ptype[t]); }
  for (auto& p : listed) ltype.push_back(typeOf(p.pod));
  for (auto& p : inTasks) ttype.push_back(typeOf(p.pod));
  const std::vector<int> pendTypes(pendSet.begin(), pendSet.end());

  // ---- key sets and domains ----
  std::map<std::vector<std::string>, uint32_t> keysetID;
  auto keysetOf = [&](std::vector<std::string> keys) -> uint32_t {
    std::sort(keys.begin(), keys.end());
    keys.erase(std::unique(keys.begin(), keys.end()), keys.end());
    for (auto& k : keys)
      if (k.empty()) throw Unsupported("a required pod (anti)affinity term with an empty topologyKey (an error in the reference, predicates.go:1311-1313)");
    auto it = keysetID.find(keys);
    if (it != keysetID.end()) return it->second;
    const uint32_t s = (uint32_t)keysetID.size();
    keysetID.emplace(keys, s);
    std::map<std::vector<std::string>, int32_t> vals;
    for (uint32_t n = 0; n < N; ++n) {
      const api::Node& node = *ssn.Nodes.at(f.nodeNames[n])->node;
      std::vector<std::string> v;
      bool ok = true;
      for (auto& k : keys) { auto l = node.Labels.find(k); if (l == node.Labels.end()) { ok = false; break; } v.push_back(l->second); }
      pa.node_domain.push_back(ok ? vals.emplace(v, (int32_t)vals.size()).first->second : -1);
    }
    pa.keyset_domains.push_back((uint32_t)vals.size());
    return s;
  };

  // ---- predicate groups ----
  struct Group { uint32_t keyset; std::vector<bool> member; };   // member: by pod type
  std::vector<Group> groups;
  std::map<std::string, uint32_t> groupID;
  auto addGroup = [&](const std::string& key, uint32_t keyset, const std::function<bool(const api::Pod&)>& member) {
    auto it = groupID.find(key);
    if (it != groupID.end()) return it->second;
    const uint32_t g = (uint32_t)groups.size();
    groupID.emplace(key, g);
    Group gr{keyset, std::vector<bool>(reps.size())};
    for (size_t ty = 0; ty < reps.size(); ++ty) gr.member[ty] = member(*reps[ty]);
    groups.push_back(std::move(gr));
    return g;
  };
  std::map<int, std::set<uint32_t>> forbid;           // pending type -> the groups it forbids
  std::map<int, int32_t> need;
  std::map<int, bool> selfMatch;
  for (int ty : pendTypes) need[ty] = -1;
  // (A) required anti-affinity terms pods own: satisfiesExistingPodsAntiAffinity (predicates.go:1400-1439)
  std::set<int> owners(ltype.begin(), ltype.end());
  owners.insert(pendTypes.begin(), pendTypes.end());
  for (int oty : owners) {
    const api::Pod& owner = *reps[oty];
    for (auto& term : requiredTerms(owner, true)) {
      if (term.TopologyKey.empty()) continue;         // node.Labels[""] never exists: the term rejects nothing (:1366)
      const TermProps props = propsOf(owner, term);
      std::vector<int> victims;
      for (int ty : pendTypes) if (props.matches(*reps[ty])) victims.push_back(ty);
      if (victims.empty()) continue;
      const uint32_t ks = keysetOf({term.TopologyKey});
      const std::string topo = term.TopologyKey, pkey = props.key;
      const uint32_t g = addGroup("A|" + pkey + "|" + topo, ks, [&](const api::Pod& x) {
        for (auto& t : requiredTerms(x, true)) {
          if (t.TopologyKey != topo) continue;
          try { if (propsOf(x, t).key == pkey) return true; } catch (const std::runtime_error&) {}   // an invalid term is no such term
        }
        return false;
      });
      for (int ty : victims) forbid[ty].insert(g);
    }
  }
  // (B) the pending pods' own required terms: satisfiesPodsAffinityAntiAffinity, slow path (:1516-1562)
  for (int ty : pendTypes) {
    const api::Pod& pod = *reps[ty];
    for (bool anti : {false, true}) {
      const auto& ts = requiredTerms(pod, anti);
      if (ts.empty()) continue;
      std::vector<TermProps> props;
      std::vector<std::string> keys, pkeys;
      for (auto& t : ts) { props.push_back(propsOf(pod, t)); pkeys.push_back(props.back().key); keys.push_back(t.TopologyKey); }
      const uint32_t ks = keysetOf(keys);
      std::sort(pkeys.begin(), pkeys.end());
      auto all = [&props](const api::Pod& x) {        // podMatchesAllAffinityTermProperties (metadata.go:601-612)
        for (auto& p : props) if (!p.matches(x)) return false;
        return true;
      };
      std::string gkey = "B|";
      for (auto& k : pkeys) gkey += k + '\x02';
      const uint32_t g = addGroup(gkey + "|" + std::to_string(ks), ks, all);
      if (anti) forbid[ty].insert(g);
      else { need[ty] = (int32_t)g; selfMatch[ty] = all(pod); }   // targetPodMatchesAffinityOfPod(pod, pod)
    }
  }
  if (groups.size() > KB_MAX_AFF_GROUPS)
    throw Unsupported(std::to_string(groups.size()) + " inter-pod affinity counter groups: more than KB_MAX_AFF_GROUPS (" + std::to_string(KB_MAX_AFF_GROUPS) + ")");
  if (keysetID.size() > 64) throw Unsupported(std::to_string(keysetID.size()) + " topology key sets: more than 64");
  const uint32_t NG = (uint32_t)groups.size();
  pa.n_groups = NG;
  std::vector<uint32_t> gOff(NG + 1, 0);
  for (uint32_t g = 0; g < NG; ++g) { pa.group_keyset.push_back(groups[g].keyset); gOff[g + 1] = gOff[g] + pa.keyset_domains[groups[g].keyset]; }
  pa.group_count0.assign(std::max(1u, gOff[NG]), 0);
  pa.group_total0.assign(std::max(1u, NG), 0);
  for (size_t i = 0; i < listed.size(); ++i) {
    for (uint32_t g = 0; g < NG; ++g) {
      if (!groups[g].member[ltype[i]]) continue;
      pa.member_groups[listed[i].pod].push_back(g);
      pa.group_total0[g]++;
      const int32_t d = pa.node_domain[(size_t)groups[g].keyset * N + listed[i].node];
      if (d >= 0) pa.group_count0[gOff[g] + d]++;
    }
  }

  // ---- priority: weights between pod types (processPod, interpod_affinity.go:119-171), kinds, per-task lists ----
  auto weights = [&](const api::Pod& in, const api::Pod& ex) {
    std::map<std::string, int64_t> w;
    auto add = [&](const api::Pod& owner, const api::PodAffinityTerm& term, const api::Pod& check, int64_t v) {
      if (term.TopologyKey.empty() || v == 0) return;   // NodesHaveSameTopologyKey is false for an empty key
      try { if (propsOf(owner, term).matches(check)) w[term.TopologyKey] += v; } catch (const std::runtime_error&) {}
    };
    for (auto& t : preferredTerms(in, false)) add(in, t.PodAffinityTerm, ex, t.Weight);
    for (auto& t : preferredTerms(in, true)) add(in, t.PodAffinityTerm, ex, -(int64_t)t.Weight);
    for (auto& t : requiredTerms(ex, false)) add(ex, t, in, 1);   // hardPodAffinityWeight = v1.DefaultHardPodAffinitySymmetricWeight (nodeorder.go:159)
    for (auto& t : preferredTerms(ex, false)) add(ex, t.PodAffinityTerm, in, t.Weight);
    for (auto& t : preferredTerms(ex, true)) add(ex, t.PodAffinityTerm, in, -(int64_t)t.Weight);
    for (auto it = w.begin(); it != w.end();) it = it->second == 0 ? w.erase(it) : std::next(it);
    return w;
  };
  std::map<std::pair<int, int>, std::map<std::string, int64_t>> wtab;
  for (int pt : pendTypes) for (size_t xt = 0; xt < reps.size(); ++xt) wtab[{pt, (int)xt}] = weights(*reps[pt], *reps[xt]);
  std::map<std::pair<std::vector<std::map<std::string, int64_t>>, bool>, int32_t> kindID;
  std::vector<int> kindRep;
  auto kindOf = [&](int xt, bool unbound) -> int32_t {
    std::vector<std::map<std::string, int64_t>> vec;
    bool nonzero = false;
    for (int pt : pendTypes) { vec.push_back(wtab[{pt, xt}]); nonzero = nonzero || !vec.back().empty(); }
    if (!nonzero) return -1;
    auto ins = kindID.emplace(std::make_pair(vec, unbound), (int32_t)kindRep.size());
    if (ins.second) { kindRep.push_back(xt); pa.kind_unbound.push_back(unbound ? 1 : 0); }
    return ins.first->second;
  };
  std::vector<int32_t> xkind;
  for (size_t i = 0; i < inTasks.size(); ++i) xkind.push_back(kindOf(ttype[i], inTasks[i].unbound));
  std::map<int, int32_t> pkind;
  for (int ty : pendTypes) pkind[ty] = kindOf(ty, true);   // a task placed in this session keeps an empty Spec.NodeName
  pa.n_kinds = (uint32_t)kindRep.size();
  pa.node_kind_count0.assign((size_t)std::max(1u, pa.n_kinds) * std::max(1u, N), 0);
  for (size_t i = 0; i < inTasks.size(); ++i) if (xkind[i] >= 0) pa.node_kind_count0[(size_t)xkind[i] * N + inTasks[i].node]++;
  struct WEntry { int32_t kind, keyset; int64_t value; };
  std::map<int, std::vector<WEntry>> wlist;
  for (int pt : pendTypes)
    for (uint32_t k = 0; k < pa.n_kinds; ++k)
      for (auto& kv : wtab[{pt, kindRep[k]}]) wlist[pt].push_back({(int32_t)k, (int32_t)keysetOf({kv.first}), kv.second});   // keys ascending
  if (keysetID.size() > 64) throw Unsupported(std::to_string(keysetID.size()) + " topology key sets: more than 64");
  pa.n_keysets = (uint32_t)keysetID.size();

  // ---- per task ----
  pa.task_forbid.assign(std::max(1u, T), 0); pa.task_contrib.assign(std::max(1u, T), 0);
  pa.task_need.assign(std::max(1u, T), -1); pa.task_kind.assign(std::max(1u, T), -1);
  pa.task_weight_off.assign(T + 1, 0);
  if (NG > 64) pa.task_xgroup_off.assign(T + 1, 0);
  for (uint32_t t = 0; t < T; ++t) {
    const int ty = ptype[t];
    pa.task_need[t] = need[ty];
    pa.task_kind[t] = pkind[ty];
    const std::set<uint32_t>& fb = forbid[ty];
    for (uint32_t g = 0; g < NG; ++g) {               // groups < 64: bits of the masks; the others: entries of task_xgroup, ascending
      const bool fg = fb.count(g) != 0, cg = groups[g].member[ty];
      if (g < 64) {
        if (fg) pa.task_forbid[t] |= 1ull << g;
        if (cg) pa.task_contrib[t] |= 1ull << g;
        continue;
      }
      if (fg || cg) pa.task_xgroup.push_back((g << 2) | (fg ? KB_XGROUP_FORBID : 0u) | (cg ? KB_XGROUP_CONTRIB : 0u));
    }
    if (!pa.task_xgroup_off.empty()) pa.task_xgroup_off[t + 1] = (uint32_t)pa.task_xgroup.size();
    for (auto& e : wlist[ty]) { pa.weight_kind.push_back(e.kind); pa.weight_keyset.push_back(e.keyset); pa.weight_value.push_back(e.value); }
    pa.task_weight_off[t + 1] = (uint32_t)pa.weight_kind.size();
    if (hasPodAffinity(*f.tasks[t]->pod)) f.task_flags[t] |= KB_TASK_HAS_POD_AFFINITY;
    if (selfMatch[ty]) f.task_flags[t] |= KB_TASK_AFF_SELF_MATCH;
  }
  // the arrays the engine reads need one element even when empty
  if (pa.node_domain.empty()) pa.node_domain.assign(std::max(1u, N), 0);
  if (pa.keyset_domains.empty()) pa.keyset_domains.push_back(0);
  if (pa.group_keyset.empty()) pa.group_keyset.push_back(0);
  if (pa.kind_unbound.empty()) pa.kind_unbound.push_back(0);
  if (pa.weight_kind.empty()) { pa.weight_kind.push_back(0); pa.weight_keyset.push_back(0); pa.weight_value.push_back(0); }
  if (pa.task_xgroup.empty()) pa.task_xgroup.push_back(0);
}

// One action on the GPU: flatten the session as it is NOW -> kb_session_load -> kb_allocate | kb_backfill -> replay the
// decisions through the session's own Allocate / Pipeline.  Every action flattens afresh, so "allocate, backfill" (the
// default list, pkg/scheduler/util.go:31-42) is two such calls, exactly like the reference runs two Execute()s on one
// session.  (A shim that wants to save the second flatten + upload can call kb_allocate and kb_backfill back to back on
// one loaded session instead: see INTEGRATION.md.)
// The session's tiers as kb_plugin_conf.  Only built-in registrations can be honoured.  `conf` points into this object,
// which therefore stays where it was built.
struct PluginConf {
  std::vector<kb_plugin_option> opts; std::vector<kb_tier> tiers; std::vector<std::vector<const char*>> keys, vals;
  kb_plugin_conf conf{};
  explicit PluginConf(const framework::Session& ssn) {
    size_t total = 0; for (auto& t : ssn.Tiers) total += t.Plugins.size();
    opts.reserve(total); keys.reserve(total); vals.reserve(total);
    for (auto& t : ssn.Tiers) {
      kb_tier ct{}; ct.n_plugins = (uint32_t)t.Plugins.size(); ct.plugins = opts.data() + opts.size();
      for (auto& p : t.Plugins) {
        auto reg = ssn.registered.find(p.Name);
        if (reg != ssn.registered.end()) for (auto b : reg->second) if (b == framework::Builtin::Foreign)
          throw std::runtime_error("plugin " + p.Name + " registered a non built-in function: the GPU path cannot honour it (no CPU fallback)");
        kb_plugin_option o{}; o.name = p.Name.c_str();
        o.enabled_job_order = p.EnabledJobOrder == 1; o.enabled_job_ready = p.EnabledJobReady == 1; o.enabled_job_pipelined = p.EnabledJobPipelined == 1;
        o.enabled_task_order = p.EnabledTaskOrder == 1; o.enabled_preemptable = p.EnabledPreemptable == 1; o.enabled_reclaimable = p.EnabledReclaimable == 1;
        o.enabled_queue_order = p.EnabledQueueOrder == 1; o.enabled_predicate = p.EnabledPredicate == 1; o.enabled_node_order = p.EnabledNodeOrder == 1;
        keys.emplace_back(); vals.emplace_back();
        for (auto& kv : p.Arguments) { keys.back().push_back(kv.first.c_str()); vals.back().push_back(kv.second.c_str()); }
        o.n_args = (uint32_t)keys.back().size(); o.arg_keys = keys.back().data(); o.arg_values = vals.back().data();
        opts.push_back(o);
      }
      tiers.push_back(ct);
    }
    conf = kb_plugin_conf{(uint32_t)tiers.size(), tiers.data()};
  }
  PluginConf(const PluginConf&) = delete;
  PluginConf& operator=(const PluginConf&) = delete;
};

// kb_snapshot over the arrays of `f` (which must outlive it)
inline kb_snapshot SnapshotOf(Flat& f) {
  kb_snapshot s{};
  s.abi_version = KB_ABI_VERSION; s.R = f.R; s.W = f.W; s.N = f.N; s.T = f.T; s.J = f.J; s.Q = f.Q;
  s.node_idle = f.node_idle.data(); s.node_releasing = f.node_releasing.data(); s.node_used = f.node_used.data(); s.node_allocatable = f.node_allocatable.data();
  s.node_alloc_present = f.node_alloc_present.data(); s.node_alloc_cpu = f.node_alloc_cpu.data(); s.node_alloc_mem = f.node_alloc_mem.data();
  s.node_nz_cpu = f.node_nz_cpu.data(); s.node_nz_mem = f.node_nz_mem.data(); s.node_pods = f.node_pods.data(); s.node_max_pods = f.node_max_pods.data();
  s.node_flags = f.node_flags.data(); s.node_labels = f.node_labels.data(); s.node_taints = f.node_taints.data(); s.node_ports = f.node_ports.data();
  s.task_initreq = f.task_initreq.data(); s.task_resreq = f.task_resreq.data(); s.task_res_present = f.task_res_present.data();
  s.task_nz_cpu = f.task_nz_cpu.data(); s.task_nz_mem = f.task_nz_mem.data(); s.task_sel_req = f.task_sel_req.data(); s.task_aff_terms = f.task_aff.data();
  s.task_n_aff_terms = f.task_n_aff.data(); s.task_tol = f.task_tol.data(); s.task_port_own = f.task_port_own.data(); s.task_port_conflict = f.task_port_conflict.data();
  s.task_flags = f.task_flags.data(); s.task_prio = f.task_prio.data(); s.task_ctime = f.task_ctime.data(); s.task_uid_rank = f.task_uid_rank.data();
  s.job_task_off = f.job_task_off.data(); s.job_min_avail = f.job_min_avail.data(); s.job_ready0 = f.job_ready0.data(); s.job_alloc0 = f.job_alloc0.data();
  s.job_alloc0_present = f.job_alloc0_present.data(); s.job_queue = f.job_queue.data(); s.job_prio = f.job_prio.data(); s.job_ctime = f.job_ctime.data();
  s.queue_weight = f.queue_weight.data(); s.queue_ctime = f.queue_ctime.data();
  s.task_n_pref_terms = f.task_n_pref.data(); s.task_pref_terms = f.task_pref.data(); s.task_pref_weights = f.task_pref_w.data();
  s.flags = f.snap_flags;
  if (f.pa.on) {
    Flat::PodAff& pa = f.pa;
    kb_pod_affinity& c = pa.c;
    c = kb_pod_affinity{};
    c.n_keysets = pa.n_keysets; c.n_groups = pa.n_groups; c.n_kinds = pa.n_kinds; c.n_weights = pa.task_weight_off[f.T];
    c.first_unbound_node = pa.first_unbound;
    c.node_domain = pa.node_domain.data(); c.keyset_domains = pa.keyset_domains.data(); c.group_keyset = pa.group_keyset.data();
    c.group_count0 = pa.group_count0.data(); c.group_total0 = pa.group_total0.data();
    c.task_forbid = pa.task_forbid.data(); c.task_need = pa.task_need.data(); c.task_contrib = pa.task_contrib.data(); c.task_kind = pa.task_kind.data();
    c.node_kind_count0 = pa.node_kind_count0.data(); c.kind_unbound = pa.kind_unbound.data(); c.task_weight_off = pa.task_weight_off.data();
    c.weight_kind = pa.weight_kind.data(); c.weight_keyset = pa.weight_keyset.data(); c.weight_value = pa.weight_value.data();
    if (!pa.task_xgroup_off.empty()) { c.task_xgroup_off = pa.task_xgroup_off.data(); c.task_xgroup = pa.task_xgroup.data(); }   // NULL when <= 64 groups
    s.pod_affinity = &c;
  }
  return s;
}

// A refusal of the engine: std::runtime_error with kb_last_error and the status
inline void Check(int rc, const char* what, kb_engine* e) {
  if (rc != KB_OK) throw std::runtime_error(std::string(what) + ": " + kb_last_error(e) + " [" + kb_status_str(rc) + "]");
}

// One engine on device 0, single GPU
struct Engine {
  kb_engine* h = nullptr;
  Engine() {
    kb_engine_opts eo{}; eo.abi_version = KB_ABI_VERSION; eo.device = 0; eo.rank = 0; eo.world_size = 1;
    Check(kb_engine_create(&eo, &h), "kb_engine_create", nullptr);
  }
  ~Engine() { if (h) kb_engine_destroy(h); }
  Engine(const Engine&) = delete;
  Engine& operator=(const Engine&) = delete;
};

// One action on the GPU: flatten the session as it is NOW -> kb_session_load -> kb_allocate | kb_backfill -> replay the
// decisions through the session's own Allocate / Pipeline.  Every action flattens afresh, so "allocate, backfill" (the
// default list, pkg/scheduler/util.go:31-42) is two such calls, exactly like the reference runs two Execute()s on one
// session.  (A shim that wants to save the second flatten + upload can call kb_allocate and kb_backfill back to back on
// one loaded session instead: see INTEGRATION.md.)
inline void ExecuteOnGpu(framework::Session* ssn, const bool backfill) {
  PluginConf pc(*ssn);
  Flat f = Flatten(*ssn);
  kb_snapshot s = SnapshotOf(f);
  Engine eng;
  Check(kb_session_load(eng.h, &s, &pc.conf), "kb_session_load", eng.h);
  std::vector<kb_decision> dec(std::max(1u, f.T));
  kb_stats st{};
  Check(backfill ? kb_backfill(eng.h, dec.data(), &st) : kb_allocate(eng.h, dec.data(), &st), backfill ? "kb_backfill" : "kb_allocate", eng.h);
  // replay in call order through the session's own Allocate / Pipeline (gang dispatch, Binder.Bind happen there)
  std::vector<uint32_t> order;
  for (uint32_t t = 0; t < f.T; ++t) if (dec[t].kind == KB_KIND_ALLOCATED || dec[t].kind == KB_KIND_PIPELINED) order.push_back(t);
  std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return dec[a].step < dec[b].step; });
  for (uint32_t t : order) {
    if (dec[t].kind == KB_KIND_ALLOCATED) ssn->Allocate(f.tasks[t], f.nodeNames[dec[t].node]);
    else ssn->Pipeline(f.tasks[t], f.nodeNames[dec[t].node]);
  }
}

class allocateAction : public framework::Action {
 public:
  std::string Name() const override { return "allocate"; }               // allocate.go:38
  // actions/allocate/allocate.go:43-194, on the GPU
  void Execute(framework::Session* ssn) override { ExecuteOnGpu(ssn, false); }
};
inline std::unique_ptr<framework::Action> New() { return std::make_unique<allocateAction>(); }

}}  // namespace actions::allocate

namespace actions { namespace backfill {
class backfillAction : public framework::Action {
 public:
  std::string Name() const override { return "backfill"; }               // backfill.go:35
  // actions/backfill/backfill.go:40-71, on the GPU
  void Execute(framework::Session* ssn) override { allocate::ExecuteOnGpu(ssn, true); }
};
inline std::unique_ptr<framework::Action> New() { return std::make_unique<backfillAction>(); }
}}  // namespace actions::backfill

// ---------------------------------------------------------------------------------------------- actions/cycle
// The configured action list ("reclaim, allocate, backfill, preempt", config/kube-batch-conf.yaml:1) as ONE kb_cycle on the
// device, handed out to the action shells: the twin of go/kbgpu/cycle.go.  The first shell that runs in a session flattens
// it as opened, loads it with its Running tasks and runs the whole list; every shell then replays only its own slice of the
// result (`bounds`) through the session's own Evict / Pipeline / Allocate and framework::Statement.  A refusal of the engine
// throws (no CPU fallback), in that shell and in every later shell of the same session.
namespace actions { namespace cycle {

// kb_running: the Running tasks of the session one by one (cycle.go::flattenRunning, builder.py meta["running"] and
// meta["running_aff_groups"]).  A task that is a member of a counter group of f.pa carries KB_RUNNING_AFF_MEMBER; its groups are
// listed in aff_group_off / aff_group, which are always filled, so the engine keeps the member bits exact when it is evicted.
struct Running {
  std::vector<std::shared_ptr<api::TaskInfo>> tasks;  // clones of the nodes' copies: what reclaim / preempt evict
  std::vector<uint32_t> node, job, present, uid_rank, flags;
  std::vector<uint32_t> aff_group_off, aff_group;     // [n+1]; the groups, with one trailing 0 so that the array is never empty
  std::vector<double> resreq;                         // [R][n]
  std::vector<int32_t> prio, waiting;                 // waiting: [J]
  std::vector<int64_t> ctime;
};

inline Running FlattenRunning(const framework::Session& ssn, const allocate::Flat& f) {
  std::map<std::string, uint32_t> jidx;
  for (uint32_t j = 0; j < f.jobIDs.size(); ++j) jidx[f.jobIDs[j]] = j;
  Running r;
  std::vector<uint32_t> nodeOf;
  for (uint32_t ni = 0; ni < f.nodeNames.size(); ++ni) {
    for (auto& kv : ssn.Nodes.at(f.nodeNames[ni])->Tasks) {
      auto& t = kv.second;
      if (t->Status != api::Running) continue;        // reclaim.go:127, preempt.go:105
      if (!jidx.count(t->Job)) continue;              // reclaim.go:131: tasks of unknown jobs are never candidates
      r.tasks.push_back(t->Clone());                  // reclaim.go:135-136: a clone, so the node's copy keeps its status
      nodeOf.push_back(ni);
    }
  }
  const uint32_t n = (uint32_t)r.tasks.size(), n1 = std::max(1u, n);
  std::vector<std::string> uids;
  for (auto& t : r.tasks) uids.push_back(t->UID);
  std::sort(uids.begin(), uids.end());
  r.node.assign(n1, 0); r.job = r.present = r.uid_rank = r.flags = r.node;
  r.resreq.assign((size_t)f.R * n1, 0); r.prio.assign(n1, 0); r.ctime.assign(n1, 0); r.aff_group_off.assign(n + 1, 0);
  for (uint32_t i = 0; i < n; ++i) {
    auto& t = *r.tasks[i];
    r.node[i] = nodeOf[i];
    r.job[i] = jidx.at(t.Job);
    allocate::resourceVec(t.Resreq, f.dims, &r.resreq[i], n, &r.present[i]);
    r.prio[i] = t.Priority;
    r.uid_rank[i] = (uint32_t)(std::lower_bound(uids.begin(), uids.end(), t.UID) - uids.begin());
    if (t.pod) {
      r.ctime[i] = t.pod->CreationTimestamp;
      const std::string& cn = t.pod->PriorityClassName;                    // conformance.go:45-53
      if (cn == "system-cluster-critical" || cn == "system-node-critical" || t.Namespace == "kube-system") r.flags[i] |= KB_RUNNING_CRITICAL;
      auto m = f.pa.member_groups.find(t.pod.get());
      if (m != f.pa.member_groups.end()) {              // its eviction takes it out of util.PodLister (kbgpu.h KB_RUNNING_AFF_MEMBER)
        r.flags[i] |= KB_RUNNING_AFF_MEMBER;
        r.aff_group.insert(r.aff_group.end(), m->second.begin(), m->second.end());
      }
    }
    r.aff_group_off[i + 1] = (uint32_t)r.aff_group.size();
  }
  r.aff_group.push_back(0);
  r.waiting.assign(std::max<size_t>(1, f.jobIDs.size()), 0);
  for (uint32_t j = 0; j < f.jobIDs.size(); ++j) {     // WaitingTaskNum (job_info.go:396-405): 0 unless an earlier action pipelined tasks
    auto& idx = ssn.Jobs.at(f.jobIDs[j])->TaskStatusIndex;
    auto it = idx.find(api::Pipelined);
    r.waiting[j] = it == idx.end() ? 0 : (int32_t)it->second.size();
  }
  return r;
}

class Cycle : public std::enable_shared_from_this<Cycle> {
 public:
  // `actions`: the configured list restricted to the four built-ins, in order.  A name may appear once: a shell finds its
  // slice of the result by its name.
  explicit Cycle(std::vector<std::string> actions) : actions_(std::move(actions)) {
    for (size_t i = 0; i < actions_.size(); ++i) {
      if (!actionID(actions_[i], nullptr)) throw std::runtime_error("kbgpu: unknown action \"" + actions_[i] + "\"");
      for (size_t k = 0; k < i; ++k) if (actions_[k] == actions_[i]) throw std::runtime_error("kbgpu: action \"" + actions_[i] + "\" is listed twice");
    }
  }
  // The four shells (framework::Action, actions/factory.go:28-33); they keep this Cycle alive
  std::vector<std::unique_ptr<framework::Action>> Actions();

  void Execute(framework::Session* ssn, const std::string& name) { ensure(ssn); replay(ssn, name); }

 private:
  static bool actionID(const std::string& name, uint8_t* id) {
    static const std::map<std::string, uint8_t> ids = {{"reclaim", KB_ACT_RECLAIM}, {"allocate", KB_ACT_ALLOCATE}, {"backfill", KB_ACT_BACKFILL}, {"preempt", KB_ACT_PREEMPT}};
    auto it = ids.find(name);
    if (it == ids.end()) return false;
    if (id) *id = it->second;
    return true;
  }
  // the whole list once per session
  void ensure(framework::Session* ssn) {
    if (uid_ == ssn->UID) { if (!failed_.empty()) throw std::runtime_error(failed_); return; }
    uid_ = ssn->UID;
    failed_.clear();
    try { run(ssn); } catch (const std::exception& e) { failed_ = e.what(); throw; }
  }
  void run(framework::Session* ssn) {
    allocate::PluginConf pc(*ssn);
    flat_ = allocate::Flatten(*ssn);
    kb_snapshot s = allocate::SnapshotOf(flat_);
    if (!engine_) engine_ = std::make_unique<allocate::Engine>();
    kb_engine* e = engine_->h;
    allocate::Check(kb_session_load(e, &s, &pc.conf), "kb_session_load", e);
    running_ = FlattenRunning(*ssn, flat_);
    Running& rf = running_;
    const uint32_t n = (uint32_t)rf.tasks.size();
    kb_running run{};
    run.n = n;
    run.node = rf.node.data(); run.job = rf.job.data(); run.resreq = rf.resreq.data(); run.res_present = rf.present.data();
    run.prio = rf.prio.data(); run.ctime = rf.ctime.data(); run.uid_rank = rf.uid_rank.data(); run.flags = rf.flags.data();
    run.job_waiting0 = rf.waiting.data();
    run.aff_group_off = rf.aff_group_off.data(); run.aff_group = rf.aff_group.data();
    // only reclaim and preempt read the Running tasks: without them a session the victim walk cannot run is not refused
    const bool evicts = std::find(actions_.begin(), actions_.end(), "reclaim") != actions_.end() ||
                        std::find(actions_.begin(), actions_.end(), "preempt") != actions_.end();
    if (evicts) allocate::Check(kb_session_load_running(e, &s, &run), "kb_session_load_running", e);
    std::vector<uint8_t> acts(actions_.size());
    for (size_t i = 0; i < actions_.size(); ++i) actionID(actions_[i], &acts[i]);
    dec_.assign(std::max(1u, flat_.T), kb_decision{});
    std::vector<uint8_t> ev(std::max(1u, n), 0);
    order_.assign(std::max(1u, n), 0);
    bounds_.assign(2 * std::max<size_t>(1, acts.size()), 0);
    kb_stats st{};
    allocate::Check(kb_cycle(e, acts.data(), (uint32_t)acts.size(), dec_.data(), ev.data(), order_.data(), bounds_.data(), &st), "kb_cycle", e);
    dec_.resize(flat_.T);
    order_.resize(n);
    evicted_.assign(n, false);
    for (uint32_t i = 0; i < n; ++i) evicted_[i] = ev[i] != 0;
  }
  // the decisions action `name` made, in the order the reference would have made the calls (cycle.go::replay)
  void replay(framework::Session* ssn, const std::string& name) {
    size_t idx = 0;
    while (idx < actions_.size() && actions_[idx] != name) ++idx;
    if (idx == actions_.size()) throw std::runtime_error("kbgpu: action \"" + name + "\" is not part of the configured cycle");
    const uint32_t lo_step = idx ? bounds_[2 * idx - 2] : 0, lo_ev = idx ? bounds_[2 * idx - 1] : 0;
    const uint32_t hi_step = bounds_[2 * idx], hi_ev = bounds_[2 * idx + 1];
    // evictions of this action, in cache.Evict order
    std::vector<uint32_t> evs;
    for (uint32_t i = 0; i < evicted_.size(); ++i) if (evicted_[i] && order_[i] >= lo_ev && order_[i] < hi_ev) evs.push_back(i);
    std::sort(evs.begin(), evs.end(), [&](uint32_t a, uint32_t b) { return order_[a] < order_[b]; });
    // placements of this action, in step order
    std::vector<uint32_t> pls;
    for (uint32_t t = 0; t < dec_.size(); ++t) {
      const kb_decision& d = dec_[t];
      if ((d.kind == KB_KIND_ALLOCATED || d.kind == KB_KIND_PIPELINED) && d.step != 0xFFFFFFFFu && d.step >= lo_step && d.step < hi_step) pls.push_back(t);
    }
    std::sort(pls.begin(), pls.end(), [&](uint32_t a, uint32_t b) { return dec_[a].step < dec_[b].step; });
    auto nodeOf = [&](uint32_t t) { return flat_.nodeNames.at((size_t)dec_[t].node); };
    if (name == "preempt") {
      // the engine only reports committed statements (preempt.go:121-131); one Statement replays them: evictions first, so
      // that node.Releasing covers the pipelined tasks (node_info.go:190-192), then Commit sends the evictions to the cache
      framework::Statement stmt(ssn);
      for (uint32_t i : evs) stmt.Evict(running_.tasks[i], "preempt");
      for (uint32_t t : pls) stmt.Pipeline(flat_.tasks[t], nodeOf(t));
      stmt.Commit();
    } else if (name == "reclaim") {
      // reclaim.go:157-185 interleaves: the victims of one reclaimer, then its Pipeline.  Replaying all evictions of the
      // action first and the pipelines after them leaves the same session state (evictions only add to Releasing).
      for (uint32_t i : evs) ssn->Evict(running_.tasks[i], "reclaim");
      for (uint32_t t : pls) ssn->Pipeline(flat_.tasks[t], nodeOf(t));
    } else {                                           // allocate, backfill
      for (uint32_t t : pls) {
        if (dec_[t].kind == KB_KIND_ALLOCATED) ssn->Allocate(flat_.tasks[t], nodeOf(t));   // dispatches when ssn.JobReady (session.go:277-285)
        else ssn->Pipeline(flat_.tasks[t], nodeOf(t));
      }
      // backfill's phantom tasks (Allocated on no node, step none: session.go:241-262) are not replayed: the reference itself
      // calls that state "will be corrected in next scheduling loop"
    }
  }

  std::vector<std::string> actions_;
  std::unique_ptr<allocate::Engine> engine_;
  std::string uid_, failed_;                           // the session the cached result belongs to; its refusal, if any
  allocate::Flat flat_;
  Running running_;
  std::vector<kb_decision> dec_;
  std::vector<bool> evicted_;
  std::vector<uint32_t> order_, bounds_;
};

// The drop-in shell of one of the four actions: same Name(), same framework::Action interface (framework/interface.go:20-32)
class action : public framework::Action {
 public:
  action(std::string name, std::shared_ptr<Cycle> cycle) : name_(std::move(name)), cycle_(std::move(cycle)) {}
  std::string Name() const override { return name_; }
  void Execute(framework::Session* ssn) override { cycle_->Execute(ssn, name_); }
 private:
  std::string name_;
  std::shared_ptr<Cycle> cycle_;
};

inline std::vector<std::unique_ptr<framework::Action>> Cycle::Actions() {
  std::vector<std::unique_ptr<framework::Action>> out;
  for (const char* name : {"reclaim", "allocate", "backfill", "preempt"}) out.push_back(std::make_unique<action>(name, shared_from_this()));
  return out;
}

// New(actions)->Actions(): a Cycle is shared by its shells
inline std::shared_ptr<Cycle> New(const std::vector<std::string>& actions) { return std::make_shared<Cycle>(actions); }

}}  // namespace actions::cycle

}  // namespace kb
