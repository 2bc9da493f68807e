/*
 * kbgpu.h — C ABI of libkbgpu.so, the H100-native engine for kube-batch's per-cycle
 * `allocate` hot path.
 *
 * The reference (kubernetes-sigs/kube-batch @ 86b2ba2, pure Go) has NO FFI boundary; the
 * boundary below is what a cgo binding inside `allocateAction.Execute`
 * (pkg/scheduler/actions/allocate/allocate.go:43-194) would call instead of running the
 * queue→job→task loop in Go.  Each entry point cites the reference code it replaces.
 *
 * Conventions: plain C, caller-allocated outputs, no torch / C++ types, return 0 on
 * success or a negative kb_status.  Never throws, never aborts.  One session in flight
 * per engine; thread-compatible, not thread-safe (matches the single `runOnce`
 * goroutine, pkg/scheduler/scheduler.go:85-102).  kb_session_load copies everything it
 * needs before returning (cgo forbids retaining Go pointers).
 *
 * There is NO CPU fallback: if no CUDA device is usable kb_engine_create fails with
 * KB_E_CUDA.
 */
#ifndef KBGPU_H_
#define KBGPU_H_

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KB_ABI_VERSION 1u

/* Compile-time capacity of the dense encodings. */
#define KB_MAX_R 8          /* resource dims: 0 = cpu (milli), 1 = memory (bytes), 2.. = scalar resources (milli) */
#define KB_MAX_W 4          /* 64-bit words per label / taint / host-port bitmask */
#define KB_MAX_PREF_TERMS 4   /* preferred node-affinity terms per task */
#define KB_MAX_AFF_TERMS 4  /* OR-ed required node-affinity terms carried per task */
#define KB_MAX_Q 256        /* queues */

typedef enum kb_status {
  KB_OK = 0,
  KB_E_BADARG = -1,
  KB_E_UNSUPPORTED_PLUGIN = -2, /* a non built-in plugin / closure the GPU path cannot honour */
  KB_E_CUDA = -3,
  KB_E_NCCL = -4,
  KB_E_STATE = -5,              /* call order violated (e.g. kb_allocate before kb_session_load) */
  KB_E_UNSUPPORTED_FEATURE = -6 /* snapshot uses a feature outside this build; kb_last_error names it (e.g. inter-pod or preferred node
                                   affinity on a sharded node axis, reclaim / preempt with inter-pod affinity beyond host-level
                                   anti-affinity, an evicted affinity group member, an action after preempt) */
} kb_status;

/* node_flags bits — evaluated once by the flattener from v1.Node
 * (vendor/k8s.io/kubernetes/pkg/scheduler/algorithm/predicates/predicates.go:1675-1698, 1633-1671). */
#define KB_NODE_NOT_READY        (1u << 0) /* a NodeReady condition with Status != True            */
#define KB_NODE_NET_UNAVAILABLE  (1u << 1) /* a NodeNetworkUnavailable condition with Status != False */
#define KB_NODE_UNSCHEDULABLE    (1u << 2) /* node.Spec.Unschedulable                               */
#define KB_NODE_MEM_PRESSURE     (1u << 3)
#define KB_NODE_DISK_PRESSURE    (1u << 4)
#define KB_NODE_PID_PRESSURE     (1u << 5)

/* task_flags bits */
#define KB_TASK_BEST_EFFORT_QOS  (1u << 0) /* v1qos.GetPodQOS(pod) == BestEffort (memory-pressure predicate only) */
#define KB_TASK_HAS_POD_AFFINITY (1u << 1) /* pod (anti)affinity terms present: needs kb_snapshot.pod_affinity, else KB_E_UNSUPPORTED_FEATURE */
#define KB_TASK_HAS_PREFERRED_NODE_AFFINITY (1u << 2) /* preferred node-affinity terms (task_pref_*)                */
#define KB_TASK_AFF_SELF_MATCH   (1u << 3) /* targetPodMatchesAffinityOfPod(pod, pod): the pod matches the namespaces + selectors of ALL its own
                                              required pod-affinity terms (vendor/.../predicates/metadata.go:767-778) — the "first pod of a
                                              series" escape of predicates.go:1545-1560                                                  */

/* kb_snapshot.flags */
#define KB_SNAPSHOT_PLACED_POD_AFFINITY (1u << 0) /* some task that is NOT pending (running / bound / allocated on a node) carries
                                                      inter-pod affinity or anti-affinity terms: the reference's predicate step 10 lets such
                                                      pods reject nodes for OTHER pods (predicates.go:1261-1288 satisfiesExistingPodsAntiAffinity)
                                                      and scores them (interpod_affinity.go:150-170): needs kb_snapshot.pod_affinity, else
                                                      KB_E_UNSUPPORTED_FEATURE                                                              */

#define KB_SNAPSHOT_LISTED_POD_WITHOUT_NODE (1u << 1) /* an AllocatedStatus task (Bound / Binding / Running / Allocated) of a session job names a
                                                      node that is NOT in ssn.Nodes (cache.Snapshot drops NotReady nodes, cache.go:633-640; the
                                                      job keeps its tasks).  util.PodLister lists the pod, CachedNodeInfo.GetNodeInfo fails
                                                      (plugins/util/util.go:93-100), and InterPodAffinityMatches returns that error for EVERY
                                                      (pod, node) pair (vendor/.../predicates.go:1381-1393): with the predicates plugin enabled
                                                      no node passes ssn.PredicateFn in this session.  The engine reproduces exactly that.      */

/* kb_decision.kind */
#define KB_KIND_NONE      0 /* task was never placed this cycle                                   */
#define KB_KIND_ALLOCATED 1 /* ssn.Allocate (framework/session.go:235)  — consumed node.Idle       */
#define KB_KIND_PIPELINED 2 /* ssn.Pipeline (framework/session.go:194)  — consumed node.Releasing  */
#define KB_KIND_SKIPPED   3 /* Resreq.IsEmpty(): skipped by allocate (allocate.go:113-118)         */

/*
 * Inter-pod (anti)affinity, flattened (SURVEY.md 8a a5 step 10 + a13).  The flattener does the string work once per snapshot:
 * it interns the topology keys the terms use, the label selectors / namespaces of the terms, and matches every pod against
 * them; the engine only counts.  Two families of counters, because the reference reads two different pod sets:
 *
 *  (P) predicate InterPodAffinityMatches (vendor/.../predicates/predicates.go:1261-1572, slow path: meta == nil) walks
 *      util.PodLister (plugins/util/util.go:37-85) = the tasks with AllocatedStatus (Bound, Binding, Running, Allocated) of the
 *      session's jobs, located by TaskInfo.NodeName.  A counter GROUP g counts such pods per topology DOMAIN of its key set:
 *        - one group per distinct required anti-affinity term an existing / pending pod owns (members: the pods owning it;
 *          key set = {term.topologyKey}); an incoming pod that matches the term's namespaces + selector FORBIDS the group
 *          (satisfiesExistingPodsAntiAffinity, :1400-1439);
 *        - one group per distinct required anti-affinity term LIST of a pending pod (members: the pods matching the namespaces +
 *          selector of ALL terms of the list, podMatchesPodAffinityTerms :1296-1320; key set = the list's topology keys — a
 *          domain is the tuple of label values): the pod FORBIDS it (:1526-1533);
 *        - one group per distinct required affinity term list of a pending pod, likewise: the pod NEEDS it — a node passes
 *          iff the group's counter of the node's domain is > 0, or no member exists anywhere and the pod matches its own terms
 *          (KB_TASK_AFF_SELF_MATCH, :1536-1560).
 *      A node whose labels lack a key of the set has domain -1 (NodesHaveSameTopologyKey is false).
 *  (S) priority CalculateInterPodAffinityPriority (vendor/.../priorities/interpod_affinity.go:99-235) walks nodeInfo.Pods() of
 *      the FEASIBLE nodes = every task in NodeInfo.Tasks whatever its status.  Pods are grouped into KINDS (same weights against
 *      every pending pod); per pending task a list of (kind, key set, weight): sum over the task's preferred (anti)affinity terms
 *      the kind matches (+-weight), the kind's required affinity terms the task matches (+1 each,
 *      v1.DefaultHardPodAffinitySymmetricWeight, nodeorder.go:159) and the kind's preferred terms the task matches (+-weight),
 *      all with that topology key.  count(n) = sum over feasible nodes m, pods on m: weight if the "pod's node" and n share the
 *      key's label value.  The "pod's node" is m for a pod whose Spec.NodeName is set; for one placed in this or an earlier
 *      session and not yet bound (Spec.NodeName == "") the reference's cachedNodeInfo.GetNodeInfo (plugins/nodeorder/nodeorder.go:
 *      49-63) returns the first node it finds holding ANY such pod — a Go map iteration; deterministic rule (SURVEY.md 8c):
 *      the lowest node index holding one (`first_unbound_node`, kept current by the engine).
 *      score = int(10 * (count - min) / (max - min)) over the feasible nodes, min and max starting at 0.
 */
#define KB_MAX_AFF_GROUPS 64
typedef struct kb_pod_affinity {
  uint32_t n_keysets;             /* distinct topology key sets                                                              */
  uint32_t n_groups;              /* <= KB_MAX_AFF_GROUPS                                                                     */
  uint32_t n_kinds;
  uint32_t n_weights;
  int32_t  first_unbound_node;    /* -1: no pod with an empty Spec.NodeName sits on a node at session open                    */
  uint32_t reserved;
  const int32_t*  node_domain;    /* [n_keysets][N] domain of node n under key set s, -1 = a key of the set is not a label of n */
  const uint32_t* keyset_domains; /* [n_keysets] number of domains                                                            */
  const uint32_t* group_keyset;   /* [n_groups]                                                                               */
  const int32_t*  group_count0;   /* groups back to back, keyset_domains[group_keyset[g]] counters each: members per domain at open */
  const int32_t*  group_total0;   /* [n_groups] members anywhere (also on nodes with domain -1)                               */
  const uint64_t* task_forbid;    /* [T] bit g: a member of g in the node's domain rejects the node for this task             */
  const int32_t*  task_need;      /* [T] group the task's required pod-affinity terms need, -1 none                          */
  const uint64_t* task_contrib;   /* [T] bit g: the task becomes a member of g once it is Allocated (not when Pipelined)      */
  const int32_t*  task_kind;      /* [T] kind the task's pod has once it sits on a node (Allocated or Pipelined), -1 = no weight anywhere */
  const int32_t*  node_kind_count0; /* [n_kinds][N] pods of kind k in NodeInfo.Tasks of node n at open                       */
  const uint8_t*  kind_unbound;   /* [n_kinds] 1: pods of the kind have an empty Spec.NodeName                                */
  const uint32_t* task_weight_off;/* [T+1] the task's entries in the three arrays below                                       */
  const int32_t*  weight_kind;    /* [n_weights]                                                                              */
  const int32_t*  weight_keyset;  /* [n_weights] a single-key key set                                                         */
  const int64_t*  weight_value;   /* [n_weights]                                                                              */
} kb_pod_affinity;

/*
 * Flattened Session snapshot (SoA).  Replaces the Go maps ssn.Jobs / ssn.Nodes / ssn.Queues
 * (framework/session.go:37-46) as input of the cycle.  All arrays are caller-owned and only
 * read during kb_session_load.
 *
 * Canonical orders (they replace Go's random map iteration, SURVEY.md §8c rules 1-4):
 *   nodes  : index == rank in ascending node Name      (allocate.go:71 GetNodeList)
 *   jobs   : index == rank in ascending JobID (UID)    (allocate.go:50)
 *   queues : index == rank in ascending QueueID (UID)
 *   tasks  : grouped by job (job_task_off); any order inside a job — the engine orders them
 *            by TaskOrderFn (session_plugins.go:318-331); task_uid_rank = rank of TaskInfo.UID.
 * Only Pending tasks are listed (allocate.go:112 iterates TaskStatusIndex[Pending]).
 */
typedef struct kb_snapshot {
  uint32_t abi_version;     /* KB_ABI_VERSION */
  uint32_t R;               /* 2..KB_MAX_R */
  uint32_t W;               /* 1..KB_MAX_W */
  uint32_t N, T, J, Q;
  uint32_t flags;           /* KB_SNAPSHOT_* */

  /* ---- nodes (api.NodeInfo, api/node_info.go:28-47) ---- */
  const double*   node_idle;          /* [R][N] NodeInfo.Idle; >= -epsilon (the cache never over-commits a node), else KB_E_BADARG */
  const double*   node_releasing;     /* [R][N] NodeInfo.Releasing                                   */
  const double*   node_used;          /* [R][N] NodeInfo.Used (bookkeeping; returned by kb_node_state) */
  const double*   node_allocatable;   /* [R][N] NodeInfo.Allocatable as float64 (drf.go:62-64, proportion.go:60-62) */
  const uint32_t* node_alloc_present; /* [N] bit r (r>=2): scalar r present in Allocatable.ScalarResources */
  const int64_t*  node_alloc_cpu;     /* [N] k8s nodeinfo allocatableResource.MilliCPU (resource_allocation.go:100-110) */
  const int64_t*  node_alloc_mem;     /* [N] k8s nodeinfo allocatableResource.Memory                 */
  const int64_t*  node_nz_cpu;        /* [N] nonzeroRequest.MilliCPU over every task in NodeInfo.Tasks (nodeinfo/node_info.go:513) */
  const int64_t*  node_nz_mem;        /* [N]                                                         */
  const int32_t*  node_pods;          /* [N] len(NodeInfo.Tasks)  (predicates.go:127)                */
  const int32_t*  node_max_pods;      /* [N] Allocatable.MaxTaskNum                                  */
  const uint32_t* node_flags;         /* [N] KB_NODE_*                                               */
  const uint64_t* node_labels;        /* [W][N] bit a: selector-requirement atom a holds on the node */
  const uint64_t* node_taints;        /* [W][N] bit a: node carries NoSchedule/NoExecute taint a     */
  const uint64_t* node_ports;         /* [W][N] bit a: host-port atom (ip,proto,port) a is in use    */

  /* ---- pending tasks (api.TaskInfo, api/job_info.go:36-54) ---- */
  const double*   task_initreq;       /* [R][T] TaskInfo.InitResreq (predicate / fit)                */
  const double*   task_resreq;        /* [R][T] TaskInfo.Resreq (bookkeeping); must be <= initreq per dim */
  const uint32_t* task_res_present;   /* [T] bit r (r>=2): scalar r present in Resreq.ScalarResources */
  const int64_t*  task_nz_cpu;        /* [T] calculatePodResourceRequest(pod, cpu) (resource_allocation.go:127) */
  const int64_t*  task_nz_mem;        /* [T]                                                         */
  const uint64_t* task_sel_req;       /* [W][T] nodeSelector atoms that must ALL hold                */
  const uint64_t* task_aff_terms;     /* [KB_MAX_AFF_TERMS][W][T] required node-affinity terms (OR of AND-masks) */
  const uint32_t* task_n_aff_terms;   /* [T] 0 = no required node affinity                           */
  const uint64_t* task_tol;           /* [W][T] taint atoms tolerated by some toleration             */
  const uint64_t* task_port_own;      /* [W][T] host-port atoms the pod occupies once placed         */
  const uint64_t* task_port_conflict; /* [W][T] host-port atoms that conflict with a wanted port (host_ports.go:96-125) */
  const uint32_t* task_flags;         /* [T] KB_TASK_*                                               */
  const int32_t*  task_prio;          /* [T] TaskInfo.Priority                                       */
  const int64_t*  task_ctime;         /* [T] Pod.CreationTimestamp (any monotone integer)            */
  const uint32_t* task_uid_rank;      /* [T] rank of TaskInfo.UID (string order), unique             */

  /* ---- jobs (api.JobInfo, api/job_info.go:127-154) ---- */
  const uint32_t* job_task_off;       /* [J+1] task range of job j                                   */
  const int32_t*  job_min_avail;      /* [J] JobInfo.MinAvailable                                    */
  const int32_t*  job_ready0;         /* [J] ReadyTaskNum() at session open (job_info.go:383)        */
  const double*   job_alloc0;         /* [R][J] sum Resreq of AllocatedStatus tasks (drf.go:71-77)   */
  const uint32_t* job_alloc0_present; /* [J] scalar presence of that sum                             */
  const uint32_t* job_queue;          /* [J] queue index                                             */
  const int32_t*  job_prio;           /* [J] JobInfo.Priority                                        */
  const int64_t*  job_ctime;          /* [J] JobInfo.CreationTimestamp                               */

  /* ---- queues (api.QueueInfo, api/queue_info.go:74-81) ---- */
  const int32_t*  queue_weight;       /* [Q]                                                         */
  const int64_t*  queue_ctime;        /* [Q]                                                         */

  /* ---- preferred node affinity (NodeAffinityPriority, vendor/.../priorities/node_affinity.go:34-77) ----
   * Only read for tasks that carry KB_TASK_HAS_PREFERRED_NODE_AFFINITY; all three may be NULL otherwise.  The CPU oracle
   * evaluates them (count = sum of the weights of the matching terms, NormalizeReduce(10) over the feasible nodes);
   * the engine evaluates them in cycle_kernel, and on the per-visit kernels (other record geometries, sessions with inter-pod terms)
   * with a pass over the feasible nodes before every visit of such a class; refused only on a sharded node axis.  preempt orders
   * its nodes with them too (the max count taken afresh for every preemptor over all nodes that pass the predicates); reclaim
   * never scores. */
  const uint32_t* task_n_pref_terms;  /* [T] 0..KB_MAX_PREF_TERMS                                    */
  const uint64_t* task_pref_terms;    /* [KB_MAX_PREF_TERMS][W][T] requirement atoms of term p: ALL must hold on the node */
  const int32_t*  task_pref_weights;  /* [KB_MAX_PREF_TERMS][T] PreferredSchedulingTerm.Weight (0 = term skipped) */

  /* ---- inter-pod (anti)affinity (predicate step 10 + InterPodAffinityPriority), NULL = no pod of the session carries terms.
   * Host-level anti-affinity (every group on a key set whose domains are the nodes, no required affinity, no live weights) is folded
   * into the node records and costs nothing; anything else runs on the per-visit kernels (fresh scan per task for the classes that
   * read the counters).  kb_session_load_running (reclaim / preempt) refuses sessions of the second kind (KB_E_UNSUPPORTED_FEATURE);
   * in the first kind the evicting actions run and only the eviction of a group MEMBER (KB_RUNNING_AFF_MEMBER) withholds the outcome. ---- */
  const kb_pod_affinity* pod_affinity;
} kb_snapshot;

/* Mirrors conf.PluginOption (pkg/scheduler/conf/scheduler_conf.go:33-56).  The Enabled* tri-states
 * are resolved by the caller: nil -> 0 (framework `isEnabled`, session_plugins.go:371) unless the
 * caller applied plugins.ApplyPluginConfDefaults (plugins/defaults.go:22-52), which sets nil -> 1. */
typedef struct kb_plugin_option {
  const char* name; /* "priority" "gang" "drf" "predicates" "proportion" "nodeorder" "conformance" */
  uint8_t enabled_job_order;
  uint8_t enabled_job_ready;
  uint8_t enabled_job_pipelined;
  uint8_t enabled_task_order;
  uint8_t enabled_preemptable;
  uint8_t enabled_reclaimable;
  uint8_t enabled_queue_order;
  uint8_t enabled_predicate;
  uint8_t enabled_node_order;
  uint32_t n_args;              /* framework.Arguments (framework/arguments.go:26) */
  const char* const* arg_keys;
  const char* const* arg_values;
} kb_plugin_option;

typedef struct kb_tier {
  uint32_t n_plugins;
  const kb_plugin_option* plugins;
} kb_tier;

typedef struct kb_plugin_conf {
  uint32_t n_tiers;
  const kb_tier* tiers;
} kb_plugin_conf;

/*
 * The Running tasks of the session, one by one: what reclaim / preempt walk (`for _, task := range n.Tasks`, reclaim.go:124-138,
 * preempt.go:195-201) and what the flattened snapshot only carries as aggregates.  Optional: only kb_reclaim / kb_preempt read it.
 * Every entry is a task with Status == Running that sits on node `node` of the snapshot and belongs to job `job`; the job's
 * job_ready0 / job_alloc0 and the node's Idle / Used / pod count already include it.
 */
#define KB_RUNNING_CRITICAL (1u << 0) /* system-cluster-critical / system-node-critical priority class or kube-system namespace (conformance.go:45-53) */
#define KB_RUNNING_AFF_MEMBER (1u << 1) /* the pod is a member of an inter-pod affinity counter group (kb_pod_affinity): evicting it takes it out of
                                            util.PodLister and can open its topology domain for other pods.  The engine keeps host-level groups as
                                            bits of the node records and does not clear them: when such a pod IS evicted (even inside a Statement that is
                                            discarded later) kb_cycle / kb_reclaim / kb_preempt return KB_E_UNSUPPORTED_FEATURE instead of a result — the
                                            shim reruns that cycle with the original actions.  Flatteners MUST set it for every Running member. */
typedef struct kb_running {
  uint32_t n;
  uint32_t reserved0;
  const uint32_t* node;         /* [n] node index                                                             */
  const uint32_t* job;          /* [n] job index                                                              */
  const double*   resreq;       /* [R][n] TaskInfo.Resreq                                                     */
  const uint32_t* res_present;  /* [n] bit r (r>=2): scalar r present in Resreq.ScalarResources               */
  const int32_t*  prio;         /* [n] TaskInfo.Priority                                                      */
  const int64_t*  ctime;        /* [n] Pod.CreationTimestamp                                                  */
  const uint32_t* uid_rank;     /* [n] rank of TaskInfo.UID among the running tasks (the reference iterates the Go map n.Tasks;
                                       the deterministic rule is UID order, SURVEY.md 8c)                     */
  const uint32_t* flags;        /* [n] KB_RUNNING_*                                                           */
  const int32_t*  job_waiting0; /* [J] or NULL (= 0): Pipelined tasks of the job at session open (WaitingTaskNum, job_info.go:396-405);
                                       non-zero only when an earlier action of the same cycle pipelined tasks  */
} kb_running;

#define KB_ENGINE_NO_OVERLAP    (1u << 0) /* never run the scan of the next visit concurrently with the replay */
#define KB_ENGINE_FORCE_OVERLAP (1u << 1) /* always (single GPU); default: only when the scan dominates (large N) */
#define KB_ENGINE_CHAIN_OFF     (1u << 2) /* one class per launch (visit_kernel); default: chained visits (single GPU, no overlap) */
#define KB_ENGINE_CHAIN2        (1u << 3) /* scan 2 classes per launch and replay the following visit from the look-ahead list  */
#define KB_ENGINE_CHAIN4        (1u << 4) /* ... 4 classes per launch                                                          */
#define KB_ENGINE_NO_PIPE       (1u << 5) /* never run the cycle as ONE persistent cooperative kernel (cycle_kernel); default: whenever
                                             the record geometry (R = 3, W = 2) and the node count fit the scanners' shared memory */
#define KB_ENGINE_SHARD         (1u << 6) /* world_size > 1: shard the node axis across the ranks (scan shard + exchange per visit).
                                             Default: every rank runs the whole cycle on the full table (replicated, no exchange):
                                             the cycle is bound by the serial replay, not by the scan */

typedef struct kb_engine_opts {
  uint32_t abi_version;     /* KB_ABI_VERSION */
  int32_t  device;          /* CUDA device ordinal */
  /* Node-axis sharding (SURVEY.md §8e).  world_size == 1: single GPU.  world_size > 1: this
   * process is rank `rank`; `nccl_unique_id` (128 bytes, from ncclGetUniqueId on rank 0,
   * distributed by the caller) bootstraps the communicator. */
  int32_t  rank;
  int32_t  world_size;
  const void* nccl_unique_id;
  uint32_t flags;           /* KB_ENGINE_* bits */
} kb_engine_opts;

typedef struct kb_decision {
  int32_t  node;          /* canonical node index, -1 if none                                  */
  uint8_t  kind;          /* KB_KIND_*                                                         */
  uint8_t  dispatched;    /* 1 if ssn.dispatch ran for the task (session.go:277-285): gang commit */
  uint16_t reserved;
  uint32_t step;          /* 0-based global order of the Allocate/Pipeline call, 0xFFFFFFFF if none */
  uint32_t dispatch_step; /* step of the Allocate call whose JobReady triggered the dispatch    */
} kb_decision;

typedef struct kb_stats {
  uint64_t pairs_logical;   /* sum over processed tasks of N  (BASELINE.md §3 work unit)        */
  uint64_t pairs_scanned;   /* (class,node) pairs the scan kernels really evaluated             */
  uint64_t pairs_replayed;  /* (task,node) pairs re-evaluated exactly during replay             */
  uint32_t tasks_processed; /* tasks popped from a task queue (allocate.go:130)                 */
  uint32_t tasks_allocated;
  uint32_t tasks_pipelined;
  uint32_t jobs_ready;      /* jobs with JobReady at cycle end that placed >= 1 task this cycle */
  uint32_t visits;          /* job visits (allocate.go:109 pops)                                */
  uint32_t kernel_launches; /* CUDA kernels launched by this kb_allocate / kb_backfill call       */
  uint32_t n_classes;       /* task equivalence classes in the session                          */
  float    gpu_ms;          /* device time of the cycle (CUDA events on the engine stream)      */
  float    load_ms;         /* host time of kb_session_load (flatten->device)                   */
  uint64_t h2d_bytes;       /* bytes kb_session_load copied host->device                        */
  uint64_t d2h_bytes;       /* bytes kb_allocate copied device->host (decisions + control block) */
  uint32_t scans;           /* visit_kernel launches that scanned the node table                */
  uint32_t rescans;         /* runs cut short because the candidate list could not certify a pick */
  uint64_t cyc_scan;        /* SM cycles (clock64) of the last CTA per launch, summed: scan phase */
  uint64_t cyc_merge;       /*   ... candidate-list merge                                        */
  uint64_t cyc_replay;      /*   ... replay + control                                            */
  uint64_t cyc_total;
  uint64_t cyc_steps;       /*   ... of cyc_replay: the per-task step loops                      */
  uint64_t cyc_ctl;         /*   ... of cyc_replay: the control plane (after_run)                 */
  uint32_t predictions;     /* overlap mode: launches whose scan ran ahead on a predicted class   */
  uint32_t mispredictions;  /*   ... of which the prediction was wrong (that launch's scan is redone) */
  uint32_t exchange_mode;   /* 0 single GPU, 1 NCCL all-gather per scan, 2 fused peer-memory exchange, 3 replicated (no exchange) */
  uint32_t chain_hits;      /* chained visits: visits replayed from a look-ahead list of an earlier launch's scan */
  uint32_t pipeline;        /* 1: the cycle ran as one persistent cooperative kernel (cycle_kernel)         */
  uint32_t pipe_requests;   /*   scan requests the replayer posted (look-ahead + urgent)                     */
  uint32_t pipe_urgent;     /*   ... of which the replayer had to wait for (no usable look-ahead list)       */
  uint32_t pipe_extends;    /*   candidate chains extended beyond the 8 pre-evaluated placement depths       */
  uint32_t pipe_patched;    /*   lists consumed with a non-empty patch set (nodes modified since the scan)   */
  uint32_t pipe_patch_entries; /* log entries re-evaluated by those patches                                  */
  uint32_t evictions;       /* kb_reclaim / kb_preempt: cache.Evict calls                                            */
  uint32_t evict_sweeps;    /*   node sweeps executed (identical failing sweeps of one job are skipped)              */
  uint64_t cyc_ring;        /* cycle_kernel, KB_PIPE_TIMING=1: main-warp cycles from the end of the runs to the write-back command (hot ring) */
  uint64_t cyc_plan;        /*   ... and in the planner (scan requests for the next visits)                           */
} kb_stats;

/* Replaces nothing in the reference (process start-up): binds a CUDA device, creates the stream,
 * and (world_size > 1) the NCCL communicator used for the per-run best-candidate exchange. */
int kb_engine_create(const kb_engine_opts* opts, struct kb_engine** out);
/* Fills `out128` (128 bytes) with a fresh ncclUniqueId (rank 0 calls it, the caller distributes it to the
 * other ranks' kb_engine_opts.nccl_unique_id).  NCCL is dlopen'ed on first use: single-GPU use never needs it. */
int kb_nccl_unique_id(void* out128);
void kb_engine_destroy(struct kb_engine* e);

/* Replaces framework.OpenSession's in-memory wiring (framework/framework.go:30-52): the snapshot
 * deep copy (cache/cache.go:627-683) arrives flattened, plugins are identified BY NAME + arguments
 * (plugins/factory.go:31-42) and their OnSessionOpen precomputation (drf.go:60-83,
 * proportion.go:58-154) is redone here.  Unknown plugin names -> KB_E_UNSUPPORTED_PLUGIN. */
int kb_session_load(struct kb_engine* e, const kb_snapshot* snap, const kb_plugin_conf* conf);

/* Replaces allocateAction.Execute (actions/allocate/allocate.go:43-194) and everything it calls
 * (util.PredicateNodes / PrioritizeNodes / SelectBestNode, ssn.Allocate / ssn.Pipeline bookkeeping,
 * JobReady gang commit).  `out` has T entries indexed like the snapshot's tasks.  The Go shim then
 * replays `out` in `step` order through the unchanged ssn.Allocate / ssn.Pipeline. */
int kb_allocate(struct kb_engine* e, kb_decision* out, kb_stats* stats);

/* Replaces backfillAction.Execute (actions/backfill/backfill.go:40-71), the action that follows allocate in the
 * default action list ("allocate, backfill", pkg/scheduler/util.go:31-42): every Pending task whose InitResreq is
 * empty (best effort) goes to the FIRST node — canonical node order, SURVEY.md §8c — on which ssn.PredicateFn passes
 * and ssn.Allocate succeeds (NodeInfo.AddTask: Resreq <= Idle, node_info.go:161-167); jobs in JobID order, tasks in UID
 * order.  Runs on the CURRENT device state: after kb_allocate it continues that cycle (step numbers, counters and the
 * gang commit carry on; a job that backfill makes ready gets its earlier Allocated tasks dispatched at that step);
 * straight after kb_session_load it is the action list "backfill" alone.  kb_allocate restarts from the loaded state.
 * `out` (T entries) is the full decision table; best-effort tasks that found no node change from SKIPPED to NONE. */
int kb_backfill(struct kb_engine* e, kb_decision* out, kb_stats* stats);

/* Hands the Running tasks of the loaded session to the engine (call after kb_session_load, before kb_reclaim / kb_preempt).
 * `snap` must be the snapshot the preceding kb_session_load was given (task order keys and job ranges are read from it again).
 * Replaces nothing in the reference: NodeInfo.Tasks is part of the session there. */
int kb_session_load_running(struct kb_engine* e, const kb_snapshot* snap, const kb_running* running);

/* Replaces reclaimAction.Execute (actions/reclaim/reclaim.go:41-193): queues by QueueOrderFn, per queue the best job by JobOrderFn
 * and its first Pending task by TaskOrderFn; the first node (canonical order) on which ssn.PredicateFn passes and the Running tasks
 * of OTHER queues that ssn.Reclaimable returns (session_plugins.go:80-118) cover InitResreq: those are evicted (ssn.Evict,
 * session.go:317-353) until InitResreq is covered and the task is pipelined there (ssn.Pipeline).  Runs from the LOADED state.
 *   out         [T]          kind PIPELINED + node + step for reclaimers, NONE otherwise
 *   evicted     [running.n]  1 if cache.Evict was called for the running task (may be NULL)
 *   evict_order [running.n]  0-based order of that call, 0xFFFFFFFF if none (may be NULL)                                  */
int kb_reclaim(struct kb_engine* e, kb_decision* out, uint8_t* evicted, uint32_t* evict_order, kb_stats* stats);

/* Replaces preemptAction.Execute (actions/preempt/preempt.go:43-270): per queue, preemption between the jobs of the queue under a
 * framework.Statement (statement.go: Evict / Pipeline, Commit when ssn.JobPipelined, Discard otherwise), then between the tasks
 * of each job; nodes in util.SortNodes order (best NodeOrderFn score first), victims by ssn.Preemptable, lowest priority first.
 * Same outputs as kb_reclaim; evictions of discarded statements are not reported (they never reached the cache).            */
int kb_preempt(struct kb_engine* e, kb_decision* out, uint8_t* evicted, uint32_t* evict_order, kb_stats* stats);

/* kb_cycle action ids: the reference's action names (actions/factory.go:28-33) */
#define KB_ACT_RECLAIM  0
#define KB_ACT_ALLOCATE 1
#define KB_ACT_BACKFILL 2
#define KB_ACT_PREEMPT  3

/* One scheduling cycle on ONE session: the configured actions one after the other from the loaded state, like
 * scheduler.go:88-101 runs `for _, action := range actions { action.Execute(ssn) }` (shipped configuration: "reclaim,
 * allocate, backfill, preempt", config/kube-batch-conf.yaml:1).  Every action sees what the previous ones left: node
 * Idle / Releasing, job / queue accounting of the plugins (drf, proportion, gang), the tasks still Pending, the Running
 * tasks not yet evicted; each action fills its own queues from that state.  At most one allocate and one backfill per list.
 *   out         [T]               the final decision table (kind / node / step; dispatched + dispatch_step from the gang commit)
 *   evicted / evict_order         as kb_reclaim, over the whole cycle (NULL when no kb_running was loaded)
 *   bounds      [2 * n_actions]   bounds[2i] = first step number NOT produced by actions 0..i, bounds[2i+1] = likewise for the
 *                                 eviction order: which action made which decision (may be NULL)                              */
int kb_cycle(struct kb_engine* e, const uint8_t* actions, uint32_t n_actions, kb_decision* out, uint8_t* evicted,
             uint32_t* evict_order, uint32_t* bounds, kb_stats* stats);

/* Bind fan-out (SURVEY.md 8f-3): the (task, node) pairs that reach cache.Bind in the cycle just run (kb_allocate / kb_backfill /
 * kb_cycle), in the order ssn.dispatch issues them (framework/session.go:277-314; among the tasks one ssn.JobReady releases at
 * once — a Go map iteration in the reference — Allocate order).  Compacted and radix-sorted on the device.  A shim hands the list
 * to ONE batched Binder call instead of a goroutine + API call per task (cache/cache.go:491-535).
 *   task, node  [T] caller-allocated; *n receives the number of binds                                                        */
int kb_bind_list(struct kb_engine* e, uint32_t* task, int32_t* node, uint32_t* n);

/* Debug / parity: predicate + score of tasks [task_lo, task_hi) against every node in the CURRENT
 * device state (util.PredicateNodes + util.PrioritizeNodes for a task range, scheduler_helper.go:63-171).
 * fit   [(task_hi-task_lo)][N] uint8 (1 = predicateFn returned nil), may be NULL
 * score [(task_hi-task_lo)][N] double (HostPriority.Score; 0 where !fit), may be NULL */
int kb_predicate_score(struct kb_engine* e, uint32_t task_lo, uint32_t task_hi, uint8_t* fit, double* score);

/* K1+K2+K3 in one launch over the whole task range: per task the packed best key
 * (score << 32 | 0xFFFFFFFF - node) against the CURRENT device state, 0 if no node fits
 * (util.SelectBestNode with the deterministic first-max rule, scheduler_helper.go:188-208). */
int kb_best_nodes(struct kb_engine* e, uint32_t task_lo, uint32_t task_hi, uint64_t* best_key);

/* Device time (CUDA events on the engine stream) of the most recent kb_predicate_score / kb_best_nodes kernel. */
int kb_last_kernel_ms(struct kb_engine* e, float* ms);

/* Current node bookkeeping after kb_allocate (NodeInfo.Idle/Releasing/Used, pod count, nonzero
 * request, used host ports) — what node_info.go:172-212 AddTask left behind.  Any pointer may be NULL. */
int kb_node_state(struct kb_engine* e, double* idle /*[R][N]*/, double* releasing /*[R][N]*/, double* used /*[R][N]*/,
                  int32_t* pods /*[N]*/, int64_t* nz_cpu /*[N]*/, int64_t* nz_mem /*[N]*/, uint64_t* ports /*[W][N]*/);

/* Job / queue ordering state at cycle end (drf.go:161-171 share, proportion.go:241-253 share + deserved). */
int kb_order_state(struct kb_engine* e, double* job_share /*[J]*/, int32_t* job_ready /*[J]*/, double* queue_share /*[Q]*/,
                   double* queue_deserved /*[R][Q]*/, double* queue_allocated /*[R][Q]*/);

const char* kb_last_error(struct kb_engine* e);
const char* kb_status_str(int status);
/* "libkbgpu <version> sm_90a" — also proves which shared object is loaded. */
const char* kb_version(void);

#ifdef __cplusplus
}
#endif
#endif /* KBGPU_H_ */
