// kb_engine.cu — libkbgpu.so: the C ABI of include/kbgpu.h over the sm_90a kernels.
//
// kb_session_load   flattens the caller's SoA snapshot into the device layout:
//                     * node table -> TMA tiles [tile][column][128 nodes]  (kb_ctl.h tile_col_*)
//                     * pending tasks -> equivalence classes (ClassRec) + per-job TaskOrderFn order
//                     * built-in plugins resolved BY NAME into EvalConf / order chains; drf and
//                       proportion OnSessionOpen precomputation redone on the host
//                     * the first `queues.Pop()` .. `jobs.Pop()` is taken on the host so the device
//                       starts with a ready run descriptor
// kb_allocate       restores the pristine mutable slab (D2D), then pumps visit_kernel launches until
//                   Ctl.done, runs the gang-commit prefix scan and copies the decisions back.
// No CPU fallback exists: every decision is produced by the kernels.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <unistd.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

#include "kb_build.h"
#include "kb_evict_build.h"
#include "kb_kernels.cuh"
#include "kb_pipe.cuh"
#include "kb_evict_launch.h"
#include "kb_bind.h"

using namespace kb;

#define KB_VERSION_STRING "libkbgpu 0.1.0 sm_90a"

namespace {

// ---- NCCL through dlopen (libnccl.so.2; prototypes per nccl.h 2.27) ----
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
struct NcclApi {
  void* h = nullptr;
  int (*GetUniqueId)(ncclUniqueId*) = nullptr;
  int (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  int (*CommDestroy)(ncclComm_t) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int /*ncclDataType_t*/, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  std::string err;
  bool load() {
    if (h) return true;
    h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) { err = std::string("dlopen libnccl.so.2: ") + dlerror(); return false; }
    GetUniqueId = (decltype(GetUniqueId))dlsym(h, "ncclGetUniqueId");
    CommInitRank = (decltype(CommInitRank))dlsym(h, "ncclCommInitRank");
    CommDestroy = (decltype(CommDestroy))dlsym(h, "ncclCommDestroy");
    AllGather = (decltype(AllGather))dlsym(h, "ncclAllGather");
    GetErrorString = (decltype(GetErrorString))dlsym(h, "ncclGetErrorString");
    if (!GetUniqueId || !CommInitRank || !CommDestroy || !AllGather || !GetErrorString) { err = "libnccl.so.2 lacks a required symbol"; h = nullptr; return false; }
    return true;
  }
};
NcclApi g_nccl;
constexpr int kNcclUint64 = 5;   // ncclUint64 (nccl.h)

}  // namespace

constexpr uint32_t KB_DEFAULT_CHAIN = 1;      // default classes per launch on one GPU (flags / env KB_CHAIN override)

struct kb_engine {
  ncclComm_t comm = nullptr;
  // peer-memory exchange (world > 1): this rank's region and every rank's region as mapped here
  uint64_t* p2p_local = nullptr;
  uint64_t* p2p_peer[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  bool p2p = false;
  unsigned char* d_xchg = nullptr;     // small device scratch for handle exchange / barriers
  int device = 0;
  int rank = 0, world = 1;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  std::string err;
  bool loaded = false;

  // session
  uint32_t R = 0, W = 0, N = 0, T = 0, J = 0, Q = 0, C = 0, NT = 0, ncols = 0, To = 0;
  unsigned char* d_mut = nullptr;      // mutable slab (current state)
  unsigned char* d_pristine = nullptr; // copy of the mutable slab as loaded
  unsigned char* d_imm = nullptr;      // immutable slab
  size_t mut_bytes = 0, imm_bytes = 0;
  DevSession dev{};                    // device pointers (allocate view)
  DevSession dev_bf{};                 // backfill view of the same slabs (kb_backfill)
  BuiltSession built;                  // host-side build of the current session
  uint32_t Tb = 0;                     // backfill order slots
  bool allocate_ran = false;           // kb_allocate ran since kb_session_load (kb_backfill continues its counters)
  uint32_t* d_task_class = nullptr;    // [T] (immutable slab)
  int32_t* d_job_ready0 = nullptr;     // [J] (immutable slab)
  Ctl* h_ctl = nullptr;                // pinned
  kb_decision* h_dec = nullptr;        // pinned [T]
  std::vector<int32_t> job_min_avail_host;
  uint32_t gang_ready = 0;
  uint32_t scan_grid = 1;
  size_t visit_smem = 0, tile_smem = 0, replay_smem = 0, chain_smem = 0;
  float load_ms = 0;
  float last_kernel_ms = 0;
  int sm_count = 132;                       // H100 SXM; replaced by the device's multiProcessorCount
  int overlap_mode = -1;
  bool pdl = true;                          // programmatic dependent launch of the visit chain (KB_PDL=0 disables)
  uint32_t kchain_req = KB_DEFAULT_CHAIN;   // classes per launch requested (flags / KB_CHAIN), 1 = visit_kernel
  bool pipe_req = true;                     // persistent pipeline (cycle_kernel) when the session's geometry allows it
  bool shard_req = false;                   // world > 1: shard the node axis (per-launch kernels + exchange) instead of replicating
  bool replicated = false;                  // world > 1 and every rank runs the whole cycle on the full node table
  bool coop_ok = false;                     // device supports cooperative launches
  size_t pipe_smem = 0;
  // reclaim / preempt (kb_evict.h): the Running tasks and the actions' own state, loaded by kb_session_load_running
  EvictBuilt ev_built;
  EvictDev ev{};
  unsigned char* d_ev_imm = nullptr; unsigned char* d_ev_mut = nullptr; unsigned char* d_ev_pristine = nullptr;
  size_t ev_cap_imm = 0, ev_cap_mut = 0;
  bool running_loaded = false;
  bool imm_dirty = false;                   // a kb_cycle rewrote parts of d_imm (job lists / order slots): re-upload before the next action from the loaded state
  uint32_t last_launches = 0;
  unsigned char* d_bind_scratch = nullptr;  // kb_bind_list: CUB temp storage + key / value double buffers
  size_t cap_bind_scratch = 0;
  int32_t* d_ready_start = nullptr;         // [J] ReadyTaskNum of every job when the cycle's allocate / backfill began (gang commit)
  size_t cap_ready_start = 0;
  uint32_t* h_dbg = nullptr;                // KB_PIPE_DEBUG=1: 64 progress words of cycle_kernel in mapped host memory
  uint32_t* d_dbg = nullptr;
  bool pipe_timing = false;                 // KB_PIPE_TIMING=1: phase timers inside cycle_kernel (kb_stats.cyc_*)
  // planner: oldest list (log entries since its stamp) accepted for the class 1 / 2 / 3 runs ahead in the queue's static order,
  // 255 = no request that far ahead (KB_PIPE_PLAN=a1,a2,a3).  0 = by session: measured on one H100 SXM (400 W), 28,16,off is best
  // with one queue (C3 45.0 ms; 40,24,off 45.6 ms; 16,8,off 46.4 ms), 10,6,off with several (C4, 8 queues: 241 ms; 16,8,off 251 ms;
  // 28,16,off 308 ms — the static order of ONE queue predicts the visit after next badly when the queues take turns)
  uint32_t pipe_plan = 0;
  double watchdog_s = 30.0;                 // a cycle_kernel that has not finished after this long is reported (with the progress words) and the process aborts: a hung cooperative kernel cannot be cancelled
  cudaGraph_t graph = nullptr;         // BATCH visit_kernel launches, captured once per distinct DevSession
  cudaGraphExec_t graph_exec = nullptr;
  uint32_t graph_launches = 0;         // kernels one launch of graph_exec runs
  DevSession graph_dev{};              // kernel parameter the graph was captured with
  size_t cap_mut = 0, cap_imm = 0, cap_dec = 0;   // capacities of the device / pinned buffers (reused across loads)
};
constexpr uint32_t BATCH = 64;

namespace {

int fail(kb_engine* e, int code, const char* fmt, ...) {
  char buf[512];
  va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
  if (e) e->err = buf;
  return code;
}
#define CUDA_TRY(e, call) do { cudaError_t _c = (call); if (_c != cudaSuccess) return fail((e), KB_E_CUDA, "%s failed: %s", #call, cudaGetErrorString(_c)); } while (0)

thread_local std::string g_create_err;

// Launch with the programmatic-stream-serialization attribute (PDL): the grid may be scheduled while its predecessor in the
// stream / captured graph is still running and blocks in griddepcontrol.wait until that one has completed and flushed.
// visit_kernel / visit_chain_kernel release their successor when only the replaying CTA is left, which hides the launch
// latency of every link of the chain behind the replay.
template <typename Kernel>
cudaError_t launch_visit(Kernel k, uint32_t grid, size_t smem, cudaStream_t st, const DevSession& D, bool pdl) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid); cfg.blockDim = dim3(SCAN_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, k, D);
}

// The per-visit launches of one link of the visit chain (allocate view, or backfill with `backfill`), in the class record type CR
// of the session.  `prepass`: the inter-pod affinity priority's passes first; `pdl`: programmatic dependent launch (graph capture).
template <class CR>
cudaError_t launch_visit_link(kb_engine* e, RecTag<CR>, const DevSession& D, const bool backfill, const bool prepass, const bool pdl) {
  if (D.aff.on) {
    // inter-pod affinity: the priority's passes over the feasible nodes (they return at once for a class without a weight
    // list), then the visit with predicate step 10 / the score term in its scan
    if (backfill) { visit_kernel<1, 1, CR><<<e->scan_grid, SCAN_THREADS, e->visit_smem, e->stream>>>(D); return cudaGetLastError(); }
    if (prepass) {
      const uint32_t ag = std::max(1u, std::min((e->N + AFF_THREADS - 1) / AFF_THREADS, (uint32_t)e->sm_count * 4u));
      const uint32_t ag1 = std::max(1u, std::min((e->N + AFF_THREADS / 32 - 1) / (AFF_THREADS / 32), (uint32_t)e->sm_count * 8u));   // pass 1: a warp per node
      aff_prepass_kernel<0, CR><<<ag, AFF_THREADS, 0, e->stream>>>(D);
      aff_prepass_kernel<1, CR><<<ag1, AFF_THREADS, 0, e->stream>>>(D);
      aff_prepass_kernel<2, CR><<<ag, AFF_THREADS, 0, e->stream>>>(D);
    }
    return launch_visit(visit_kernel<0, 1, CR>, e->scan_grid, e->visit_smem, e->stream, D, pdl);
  }
  if (backfill) { visit_kernel<1, 0, CR><<<e->scan_grid, SCAN_THREADS, e->visit_smem, e->stream>>>(D); return cudaGetLastError(); }
  if (D.overlap) { visit_overlap_kernel<CR><<<e->scan_grid + 1, SCAN_THREADS, e->visit_smem, e->stream>>>(D); return cudaGetLastError(); }
  if (D.kchain == 2) return launch_visit(visit_chain_kernel<2, CR>, e->scan_grid, e->chain_smem, e->stream, D, pdl);
  if (D.kchain == 4) return launch_visit(visit_chain_kernel<4, CR>, e->scan_grid, e->chain_smem, e->stream, D, pdl);
  return launch_visit(visit_kernel<0, 0, CR>, e->scan_grid, e->visit_smem, e->stream, D, pdl);
}

// Enqueues n links of the visit chain: the per-visit launches and, sharded without peer memory, the all-gather of every rank's top-32
// keys and node records and the identical replay.  Returns KB_OK with *kernels = the kernels enqueued, or the failure (e->err).
int enqueue_links(kb_engine* e, const DevSession& D, const bool backfill, const bool pdl, const uint32_t n, uint32_t* kernels) {
  const bool prepass = D.aff.on && !backfill && (D.aff.has_weights || D.aff.has_pref);   // nodeorder is off in backfill: no passes
  const bool gather = e->world > 1 && !D.p2p && !e->replicated;     // a replicated rank replays in visit_kernel itself (DevSession.world == 1)
  for (uint32_t i = 0; i < n; ++i) {
    CUDA_TRY(e, with_rec(e->built.rec, [&](auto t) { return launch_visit_link(e, t, D, backfill, prepass, pdl); }));
    if (gather) {
      const int rc = g_nccl.AllGather(D.sendbuf, D.recvbuf, (size_t)xchg_u64(e->ncols), kNcclUint64, e->comm, e->stream);
      if (rc != 0) return fail(e, KB_E_NCCL, "ncclAllGather: %s", g_nccl.GetErrorString(rc));
      if (backfill) replay_kernel<1><<<1, 64, e->replay_smem, e->stream>>>(D);
      else replay_kernel<0><<<1, 64, e->replay_smem, e->stream>>>(D);
    }
  }
  CUDA_TRY(e, cudaGetLastError());
  *kernels = n * ((prepass ? 4u : 1u) + (gather ? 1u : 0u));
  return KB_OK;
}

static_assert(std::is_same<ClassRec, ClassRecNarrow>::value, "RecKind::Own runs the kernels' default (narrow) instances");
// the wide and wide-atom instances' staging buffers (scan_tpi) fit next to their VisitSmem, down to the widest record at one tile
// per iteration: the scan_tpi budget and two tiles of the widest record
template <class CR>
constexpr bool visit_smem_fits() {
  return ((sizeof(VisitSmem<CR>) + 127) / 128) * 128 + std::max<size_t>(160 * 1024, 2 * (size_t)max_cols<CR>() * TILE_NODES * 8) <= 227 * 1024;
}
static_assert(visit_smem_fits<ClassRecWide>(), "wide VisitSmem + scan_tpi budget / two tiles of the widest record");
static_assert(visit_smem_fits<ClassRecAtoms>(), "wide-atom VisitSmem + scan_tpi budget / two tiles of the widest record");

// Shared-memory sizes and limits of the kernels of class record type CR for a session with B.tpi staged tiles of e->tile_smem bytes
template <class CR>
cudaError_t set_kernel_smem(kb_engine* e, RecTag<CR>, const uint32_t tpi, const uint32_t kchain) {
  e->visit_smem = ((sizeof(VisitSmem<CR>) + 127) / 128) * 128 + 2 * (size_t)tpi * e->tile_smem;
  cudaError_t c = cudaSuccess;
  for (const void* k : {(const void*)visit_kernel<0, 0, CR>, (const void*)visit_kernel<1, 0, CR>, (const void*)visit_kernel<0, 1, CR>,
                        (const void*)visit_kernel<1, 1, CR>, (const void*)visit_overlap_kernel<CR>})
    if (c == cudaSuccess) c = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)e->visit_smem);
  e->chain_smem = 0;
  if (c == cudaSuccess && kchain == 2) {
    e->chain_smem = chain_smem_header<2, CR>() + 2 * (size_t)tpi * e->tile_smem;
    c = cudaFuncSetAttribute(visit_chain_kernel<2, CR>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)e->chain_smem);
  }
  if (c == cudaSuccess && kchain == 4) {
    e->chain_smem = chain_smem_header<4, CR>() + 2 * (size_t)tpi * e->tile_smem;
    c = cudaFuncSetAttribute(visit_chain_kernel<4, CR>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)e->chain_smem);
  }
  if (c == cudaSuccess) c = cudaFuncSetAttribute(matrix_kernel<CR>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)e->tile_smem);
  if (c == cudaSuccess) c = cudaFuncSetAttribute(best_nodes_kernel<CR>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)e->tile_smem);
  return c;
}

void free_graph(kb_engine* e) {
  if (e->graph_exec) cudaGraphExecDestroy(e->graph_exec);
  if (e->graph) cudaGraphDestroy(e->graph);
  e->graph_exec = nullptr; e->graph = nullptr;
}
void free_session(kb_engine* e) {
  free_graph(e);
  e->cap_mut = e->cap_imm = e->cap_dec = 0;
  if (e->d_mut) cudaFree(e->d_mut);
  if (e->d_pristine) cudaFree(e->d_pristine);
  if (e->d_imm) cudaFree(e->d_imm);
  if (e->h_dec) cudaFreeHost(e->h_dec);
  if (e->d_ev_imm) cudaFree(e->d_ev_imm);
  if (e->d_ev_mut) cudaFree(e->d_ev_mut);
  if (e->d_ev_pristine) cudaFree(e->d_ev_pristine);
  if (e->d_ready_start) cudaFree(e->d_ready_start);
  if (e->d_bind_scratch) cudaFree(e->d_bind_scratch);
  e->d_bind_scratch = nullptr; e->cap_bind_scratch = 0;
  e->d_ready_start = nullptr; e->cap_ready_start = 0;
  e->d_ev_imm = e->d_ev_mut = e->d_ev_pristine = nullptr; e->ev_cap_imm = e->ev_cap_mut = 0; e->running_loaded = false;
  e->d_mut = e->d_pristine = e->d_imm = nullptr; e->h_dec = nullptr;
  e->loaded = false;
}

// Collective over e->comm.  Every rank allocates its exchange region, the IPC handles are all-gathered through NCCL,
// peers are opened, and the outcome is all-gathered again so that all ranks agree on p2p vs NCCL.
void setup_p2p(kb_engine* e) {
  e->p2p = false;
  const int W = e->world;
  if (W > (int)KB_MAX_WORLD) return;
  const char* off = getenv("KB_NO_P2P");
  bool ok = !(off && off[0] == '1');
  if (cudaMalloc(&e->d_xchg, 64 * 8 + 64) != cudaSuccess) return;
  if (cudaMalloc(&e->p2p_local, P2P_REGION_BYTES) != cudaSuccess) { e->p2p_local = nullptr; ok = false; }
  cudaIpcMemHandle_t mine;
  memset(&mine, 0, sizeof mine);
  if (ok) {
    cudaMemset(e->p2p_local, 0, P2P_REGION_BYTES);
    if (cudaIpcGetMemHandle(&mine, e->p2p_local) != cudaSuccess) { ok = false; cudaGetLastError(); }
  }
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
  cudaMemcpy(e->d_xchg + (size_t)e->rank * 64, &mine, 64, cudaMemcpyHostToDevice);
  if (g_nccl.AllGather(e->d_xchg + (size_t)e->rank * 64, e->d_xchg, 64, 0 /*ncclChar*/, e->comm, e->stream) != 0) return;
  if (cudaStreamSynchronize(e->stream) != cudaSuccess) return;
  cudaIpcMemHandle_t all[8];
  cudaMemcpy(all, e->d_xchg, (size_t)W * 64, cudaMemcpyDeviceToHost);
  for (int r = 0; r < W && ok; ++r) {
    if (r == e->rank) { e->p2p_peer[r] = e->p2p_local; continue; }
    void* ptr = nullptr;
    if (cudaIpcOpenMemHandle(&ptr, all[r], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { ok = false; cudaGetLastError(); break; }
    e->p2p_peer[r] = (uint64_t*)ptr;
  }
  // agree
  unsigned char st = ok ? 1 : 0;
  cudaMemcpy(e->d_xchg + 512 + e->rank, &st, 1, cudaMemcpyHostToDevice);
  if (g_nccl.AllGather(e->d_xchg + 512 + e->rank, e->d_xchg + 512, 1, 0, e->comm, e->stream) != 0) return;
  if (cudaStreamSynchronize(e->stream) != cudaSuccess) return;
  unsigned char sts[8];
  cudaMemcpy(sts, e->d_xchg + 512, (size_t)W, cudaMemcpyDeviceToHost);
  bool all_ok = true;
  for (int r = 0; r < W; ++r) all_ok = all_ok && sts[r] == 1;
  e->p2p = all_ok;
}

}  // namespace

extern "C" {

const char* kb_version(void) { return KB_VERSION_STRING; }

int kb_nccl_unique_id(void* out128) {
  if (!out128) return KB_E_BADARG;
  if (!g_nccl.load()) { g_create_err = g_nccl.err; return KB_E_NCCL; }
  ncclUniqueId id;
  int rc = g_nccl.GetUniqueId(&id);
  if (rc != 0) { g_create_err = std::string("ncclGetUniqueId: ") + g_nccl.GetErrorString(rc); return KB_E_NCCL; }
  memcpy(out128, id.internal, sizeof id.internal);
  return KB_OK;
}

const char* kb_status_str(int s) {
  switch (s) {
    case KB_OK: return "KB_OK";
    case KB_E_BADARG: return "KB_E_BADARG";
    case KB_E_UNSUPPORTED_PLUGIN: return "KB_E_UNSUPPORTED_PLUGIN";
    case KB_E_CUDA: return "KB_E_CUDA";
    case KB_E_NCCL: return "KB_E_NCCL";
    case KB_E_STATE: return "KB_E_STATE";
    case KB_E_UNSUPPORTED_FEATURE: return "KB_E_UNSUPPORTED_FEATURE";
  }
  return "KB_E_UNKNOWN";
}

const char* kb_last_error(kb_engine* e) { return e ? e->err.c_str() : g_create_err.c_str(); }

int kb_engine_create(const kb_engine_opts* opts, kb_engine** out) {
  if (!opts || !out) { g_create_err = "opts/out is NULL"; return KB_E_BADARG; }
  if (opts->abi_version != KB_ABI_VERSION) { g_create_err = "abi_version mismatch"; return KB_E_BADARG; }
  *out = nullptr;
  int ndev = 0;
  cudaError_t c = cudaGetDeviceCount(&ndev);
  if (c != cudaSuccess || ndev == 0) {
    g_create_err = std::string("no usable CUDA device (there is no CPU fallback): ") + cudaGetErrorString(c);
    return KB_E_CUDA;
  }
  if (opts->device < 0 || opts->device >= ndev) { g_create_err = "device ordinal out of range"; return KB_E_BADARG; }
  const int world = opts->world_size <= 0 ? 1 : opts->world_size;
  if (world > 1 && (opts->rank < 0 || opts->rank >= world || !opts->nccl_unique_id)) {
    g_create_err = "world_size > 1 needs 0 <= rank < world_size and a 128-byte nccl_unique_id"; return KB_E_BADARG; }
  if (world > 1 && !g_nccl.load()) { g_create_err = g_nccl.err; return KB_E_NCCL; }
  kb_engine* e = new kb_engine();
  e->device = opts->device;
  e->rank = world > 1 ? opts->rank : 0; e->world = world;
  e->overlap_mode = (opts->flags & KB_ENGINE_NO_OVERLAP) ? 0 : (opts->flags & KB_ENGINE_FORCE_OVERLAP) ? 1 : -1;
  e->kchain_req = (opts->flags & KB_ENGINE_CHAIN_OFF) ? 1u : (opts->flags & KB_ENGINE_CHAIN4) ? 4u : (opts->flags & KB_ENGINE_CHAIN2) ? 2u : KB_DEFAULT_CHAIN;
  e->pipe_req = !(opts->flags & KB_ENGINE_NO_PIPE) && e->overlap_mode != 1 && e->kchain_req == 1;
  e->shard_req = (opts->flags & KB_ENGINE_SHARD) != 0;
  if (const char* pp = getenv("KB_PIPE")) e->pipe_req = atoi(pp) != 0;
  if (const char* sh = getenv("KB_SHARD")) e->shard_req = atoi(sh) != 0;
  if (const char* pd = getenv("KB_PDL")) e->pdl = atoi(pd) != 0;
  if (const char* wd = getenv("KB_WATCHDOG_S")) e->watchdog_s = atof(wd);
  if (const char* pt = getenv("KB_PIPE_TIMING")) e->pipe_timing = atoi(pt) != 0;
  if (const char* pp = getenv("KB_PIPE_PLAN")) {
    unsigned a1 = 28, a2 = 16, a3 = 255;
    if (sscanf(pp, "%u,%u,%u", &a1, &a2, &a3) == 3 && a1 >= 1 && a1 < 256 && a2 < 256 && a3 < 256) e->pipe_plan = (a1 << 8) | (a2 << 16) | (a3 << 24);
  }
  if (const char* kc = getenv("KB_CHAIN")) { const int v = atoi(kc); if (v == 1 || v == 2 || v == 4) e->kchain_req = (uint32_t)v; }
  if ((c = cudaSetDevice(e->device)) != cudaSuccess || (c = cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking)) != cudaSuccess ||
      (c = cudaEventCreate(&e->ev0)) != cudaSuccess || (c = cudaEventCreate(&e->ev1)) != cudaSuccess ||
      (c = cudaMallocHost(&e->h_ctl, sizeof(Ctl))) != cudaSuccess) {
    g_create_err = std::string("CUDA init failed: ") + cudaGetErrorString(c);
    delete e; return KB_E_CUDA;
  }
  if (const char* dbg = getenv("KB_PIPE_DEBUG")) if (atoi(dbg) != 0) {
    if (cudaHostAlloc(&e->h_dbg, 64 * 4, cudaHostAllocMapped) == cudaSuccess && cudaHostGetDevicePointer(&e->d_dbg, e->h_dbg, 0) == cudaSuccess) memset(e->h_dbg, 0, 64 * 4);
    else { e->h_dbg = nullptr; e->d_dbg = nullptr; cudaGetLastError(); }
  }
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, e->device) == cudaSuccess) { e->sm_count = prop.multiProcessorCount; e->coop_ok = prop.cooperativeLaunch != 0; }
  if (world > 1) {
    ncclUniqueId id;
    memcpy(id.internal, opts->nccl_unique_id, sizeof id.internal);
    int rc = g_nccl.CommInitRank(&e->comm, world, id, e->rank);
    if (rc != 0) { g_create_err = std::string("ncclCommInitRank: ") + g_nccl.GetErrorString(rc); kb_engine_destroy(e); return KB_E_NCCL; }
    setup_p2p(e);      // collective; falls back to the NCCL exchange when peer memory is unavailable on any rank
  }
  *out = e;
  return KB_OK;
}

void kb_engine_destroy(kb_engine* e) {
  if (!e) return;
  cudaSetDevice(e->device);
  free_session(e);
  for (int r = 0; r < 8; ++r) if (e->p2p_peer[r] && r != e->rank) cudaIpcCloseMemHandle(e->p2p_peer[r]);
  if (e->p2p_local) cudaFree(e->p2p_local);
  if (e->d_xchg) cudaFree(e->d_xchg);
  if (e->comm) g_nccl.CommDestroy(e->comm);
  if (e->h_ctl) cudaFreeHost(e->h_ctl);
  if (e->h_dbg) cudaFreeHost(e->h_dbg);
  if (e->ev0) cudaEventDestroy(e->ev0);
  if (e->ev1) cudaEventDestroy(e->ev1);
  if (e->stream) cudaStreamDestroy(e->stream);
  delete e;
}

int kb_session_load(kb_engine* e, const kb_snapshot* s, const kb_plugin_conf* conf) {
  if (!e) return KB_E_BADARG;
  auto t_start = std::chrono::steady_clock::now();
  CUDA_TRY(e, cudaSetDevice(e->device));
  e->loaded = false;
  BuiltSession& B = e->built;        // kept across loads: the host slabs' capacity is recycled
  BuildErr be;
  uint32_t kchain = e->world == 1 ? e->kchain_req : 1u;
  {
    // the chain kernel keeps K class records, K lists and the fold buffers next to the tile staging buffers: when that
    // does not fit into shared memory for this record width, fall back to fewer classes per launch
    const uint32_t R = s ? s->R : 2, W = s ? s->W : 1;
    const size_t tile_b = (size_t)tile_ncols(R, W) * TILE_NODES * 8;
    const uint32_t tpi = scan_tpi(R, W);
    const size_t lim = 227 * 1024;
    with_rec(rec_kind(R, W), [&](auto t) {
      using CR = typename decltype(t)::type;
      if (kchain == 4 && chain_smem_header<4, CR>() + 2 * tpi * tile_b > lim) kchain = 2;
      if (kchain == 2 && chain_smem_header<2, CR>() + 2 * tpi * tile_b > lim) kchain = 1;
    });
  }
  // world > 1: by default every rank runs the whole cycle on the full (replicated) node table — the cycle is bound by the
  // serial replay, not by the scan, so sharding the scan only adds an exchange per visit (DESIGN.md §6); KB_ENGINE_SHARD
  // selects the node-sharded per-launch path instead.
  // inter-pod affinity (kb_pod_affinity): per-visit kernels on the full table; with world > 1 every rank runs the whole cycle
  // (replicated) unless KB_ENGINE_SHARD asks for the sharded path, which such sessions refuse
  const bool aff_session = s && s->pod_affinity != nullptr;
  // more resource dimensions or mask words than the sharded exchange's records carry (P2P_RANK_U64): replicated unless
  // KB_ENGINE_SHARD asks for the sharded path, which such sessions refuse (kb_build.h)
  const bool wide_session = s && rec_kind(s->R, s->W) != RecKind::Own;
  const bool pipe_ok = e->pipe_req && e->coop_ok;
  const bool pipe_try = (pipe_ok && (e->world == 1 || !e->shard_req)) || ((aff_session || wide_session) && !e->shard_req);      // = the full table on this rank
  int rc_build = build_session(s, conf, (uint32_t)std::max(1, e->sm_count), B, &be, pipe_try ? 0u : (uint32_t)e->rank,
                               pipe_try ? 1u : (uint32_t)e->world, e->overlap_mode, kchain, false, (pipe_try && pipe_ok) ? 1 : 0, true);
  if (rc_build == KB_OK && pipe_try && !B.pipe && e->world > 1 && !aff_session && !wide_session)       // geometry outside the pipeline: fall back to the sharded path
    rc_build = build_session(s, conf, (uint32_t)std::max(1, e->sm_count), B, &be, (uint32_t)e->rank, (uint32_t)e->world, e->overlap_mode, kchain,
                             false, 0, true);
  if (rc_build) return fail(e, rc_build, "%s", be.msg.c_str());
  e->replicated = e->world > 1 && B.world == 1;
  const uint32_t R = B.R, W = B.W, N = B.N, T = B.T, J = B.J, Q = B.Q, C = B.C, NT = B.NT, ncols = B.ncols, To = B.To, grid = B.grid;
  const size_t tile_u64 = (size_t)ncols * TILE_NODES;
  Slab& mut = B.mut; Slab& imm = B.imm;
  const OffImm& oi = B.oi;
  const HostConf& hc = B.hc;

  // ---------------- upload ----------------
  e->mut_bytes = mut.host.size(); e->imm_bytes = imm.host.size();
  // buffers are reused across sessions (a scheduler loads one snapshot per cycle): grow-only
  if (e->mut_bytes > e->cap_mut) {
    if (e->d_mut) cudaFree(e->d_mut);
    if (e->d_pristine) cudaFree(e->d_pristine);
    e->d_mut = e->d_pristine = nullptr; e->cap_mut = 0;
    const size_t cap = e->mut_bytes + e->mut_bytes / 4;
    CUDA_TRY(e, cudaMalloc(&e->d_mut, cap));
    CUDA_TRY(e, cudaMalloc(&e->d_pristine, cap));
    e->cap_mut = cap;
  }
  if (e->imm_bytes > e->cap_imm) {
    if (e->d_imm) cudaFree(e->d_imm);
    e->d_imm = nullptr; e->cap_imm = 0;
    const size_t cap = e->imm_bytes + e->imm_bytes / 4;
    CUDA_TRY(e, cudaMalloc(&e->d_imm, cap));
    e->cap_imm = cap;
  }
  const size_t dec_bytes = std::max<size_t>(1, T) * sizeof(kb_decision);
  if (dec_bytes > e->cap_dec) {
    if (e->h_dec) cudaFreeHost(e->h_dec);
    e->h_dec = nullptr; e->cap_dec = 0;
    CUDA_TRY(e, cudaMallocHost(&e->h_dec, dec_bytes + dec_bytes / 4));
    e->cap_dec = dec_bytes + dec_bytes / 4;
  }
  CUDA_TRY(e, cudaMemcpyAsync(e->d_pristine, mut.host.data(), e->mut_bytes, cudaMemcpyHostToDevice, e->stream));
  CUDA_TRY(e, cudaMemcpyAsync(e->d_imm, imm.host.data(), e->imm_bytes, cudaMemcpyHostToDevice, e->stream));
  CUDA_TRY(e, cudaMemcpyAsync(e->d_mut, e->d_pristine, e->mut_bytes, cudaMemcpyDeviceToDevice, e->stream));
  CUDA_TRY(e, cudaStreamSynchronize(e->stream));
  B.bind(e->dev, e->d_mut, e->d_imm);
  e->dev.p2p = (e->world > 1 && e->p2p && !e->replicated) ? 1u : 0u;
  for (int r = 0; r < 8; ++r) e->dev.peer_base[r] = e->p2p_peer[r];
  B.bind_backfill(e->dev_bf, e->d_mut, e->d_imm);
  e->dev_bf.p2p = e->dev.p2p;
  for (int r = 0; r < 8; ++r) e->dev_bf.peer_base[r] = e->p2p_peer[r];
  e->Tb = B.Tb;
  e->allocate_ran = false;
  e->running_loaded = false;
  e->imm_dirty = false;
  e->d_task_class = (uint32_t*)(e->d_imm + oi.task_class);
  e->d_job_ready0 = (int32_t*)(e->d_imm + oi.job_ready0);
  e->R = R; e->W = W; e->N = N; e->T = T; e->J = J; e->Q = Q; e->C = C; e->NT = NT; e->ncols = ncols; e->To = To;
  e->gang_ready = hc.gang_ready;
  e->job_min_avail_host = B.job_min_avail;
  e->scan_grid = grid;
  e->tile_smem = tile_u64 * 8;
  CUDA_TRY(e, with_rec(B.rec, [&](auto t) { return set_kernel_smem(e, t, B.tpi, B.kchain); }));
  // the cycle is a chain of identical launches: capture BATCH of them into one graph (one host call per batch)
  e->replay_smem = ((sizeof(VisitSmem<>) + 127) / 128) * 128;
  CUDA_TRY(e, cudaFuncSetAttribute(replay_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)e->replay_smem));
  CUDA_TRY(e, cudaFuncSetAttribute(replay_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)e->replay_smem));
  e->pipe_smem = 0;
  if (e->dev.pipe) {
    const size_t scan_b = pipe_scan_header() + (size_t)e->dev.pipe_tpc * e->tile_smem;
    e->pipe_smem = std::max(scan_b, sizeof(ReplaySmem<18>));
    CUDA_TRY(e, cudaFuncSetAttribute(cycle_kernel<3, 2, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)e->pipe_smem));
    CUDA_TRY(e, cudaFuncSetAttribute(cycle_kernel<3, 2, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)e->pipe_smem));
    int occ = 0;
    CUDA_TRY(e, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, cycle_kernel<3, 2, 1>, PIPE_THREADS, e->pipe_smem));
    if (occ < 1 || (int)e->dev.pipe_S + 1 > e->sm_count * occ)
      return fail(e, KB_E_CUDA, "cycle_kernel: %u CTAs cannot be co-resident (occupancy %d x %d SMs)", e->dev.pipe_S + 1, occ, e->sm_count);
  }
  if (!e->dev.pipe && (!e->graph_exec || memcmp(&e->graph_dev, &e->dev, sizeof(DevSession)) != 0)) {
    free_graph(e);
    // the cycle is a chain of identical launches: capture BATCH of them into one graph (one host call per batch)
    cudaError_t ce = cudaStreamBeginCapture(e->stream, cudaStreamCaptureModeThreadLocal);
    const bool pdl = e->pdl && (e->world == 1 || e->replicated);
    bool ok = ce == cudaSuccess && enqueue_links(e, e->dev, false, pdl, BATCH, &e->graph_launches) == KB_OK;
    cudaGraph_t g = nullptr;
    ce = cudaStreamEndCapture(e->stream, &g);
    ok = ok && ce == cudaSuccess && g != nullptr;
    if (ok) ok = cudaGraphInstantiate(&e->graph_exec, g, 0) == cudaSuccess;
    if (ok) { e->graph = g; memcpy(&e->graph_dev, &e->dev, sizeof(DevSession)); }
    else {
      if (g) cudaGraphDestroy(g);
      e->graph_exec = nullptr;
      cudaGetLastError();                      // clear; kb_allocate falls back to plain stream launches
      if (e->world == 1) return fail(e, KB_E_CUDA, "CUDA graph capture of the visit chain failed");
    }
  }
  e->loaded = true;
  e->load_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t_start).count();
  return KB_OK;
}

namespace {

int finish_cycle(kb_engine* e, const bool backfill, const int32_t* d_ready_start, kb_decision* out, kb_stats* stats, uint32_t launches,
                 const uint32_t batch, const bool use_pipe);

// back to the as-loaded state: the mutable slab, the evict path's mutable slab, and — when a kb_cycle re-sorted job lists or
// task order slots in it — the "immutable" slab
cudaError_t restore_session(kb_engine* e) {
  cudaError_t c = cudaMemcpyAsync(e->d_mut, e->d_pristine, e->mut_bytes, cudaMemcpyDeviceToDevice, e->stream);
  if (c == cudaSuccess && e->imm_dirty) {
    c = cudaMemcpyAsync(e->d_imm, e->built.imm.host.data(), e->imm_bytes, cudaMemcpyHostToDevice, e->stream);
    e->imm_dirty = false;
  }
  if (c == cudaSuccess && e->running_loaded)
    c = cudaMemcpyAsync(e->d_ev_mut, e->d_ev_pristine, e->ev_built.mut.host.size(), cudaMemcpyDeviceToDevice, e->stream);
  return c;
}

// One action of the cycle on view `D`: launches until the view's control block reports done, then the gang commit and
// the read-back.  allocate (D = e->dev) starts from the pristine tables and pumps the captured graph; backfill
// (D = e->dev_bf) continues on the current tables with plain launches (there are few best-effort tasks).
// in_cycle: the action continues kb_cycle's session (no restore, set-up done by the caller, no commit / read-back here)
int run_action(kb_engine* e, const bool backfill, kb_decision* out, kb_stats* stats, const bool in_cycle = false) {
  const DevSession& D = backfill ? e->dev_bf : e->dev;
  CUDA_TRY(e, cudaSetDevice(e->device));
  if (!in_cycle) {
    CUDA_TRY(e, cudaEventRecord(e->ev0, e->stream));
    if (!backfill) CUDA_TRY(e, restore_session(e));
    else seed_backfill_kernel<<<1, 32, 0, e->stream>>>(e->dev.ctl, e->dev_bf.ctl, e->allocate_ran ? 1 : 0);
  }
  if (!backfill) e->allocate_ran = true;
  if (e->world > 1 && D.p2p && !e->replicated) {
    // a new action restarts the exchange sequence at 1: clear my flags, then make sure every rank has done so before
    // anybody can raise one (the all-gather is only used as a stream-ordered barrier)
    CUDA_TRY(e, cudaMemsetAsync(e->p2p_local + P2P_FLAG_OFF, 0, 2 * KB_MAX_WORLD * 8, e->stream));
    if (g_nccl.AllGather(e->d_xchg + 520 + e->rank, e->d_xchg + 520, 1, 0, e->comm, e->stream) != 0)
      return fail(e, KB_E_NCCL, "barrier all-gather failed");
  }
  uint32_t launches = 0;
  // every visit pops one queue entry or consumes >= 1 task; rescans are bounded by tasks as well
  const uint64_t cap = (D.aff.on ? 4ull : 1ull) * (4ull * ((uint64_t)e->J + e->To + e->Tb) + 1024);
  const bool use_pipe = !backfill && D.pipe;
  const bool use_graph = !backfill && !use_pipe && e->graph_exec;
  const uint32_t batch = backfill ? 16u : BATCH;
  for (;;) {
    if (use_pipe) {
      // ONE cooperative launch runs the whole cycle: pipe_S scanner CTAs with resident tiles + the replayer CTA
      DevSession dv = D;
      dv.dbg = e->d_dbg;
      const uint32_t plan = e->pipe_plan ? e->pipe_plan : (D.Q > 1 ? ((10u << 8) | (6u << 16) | (255u << 24)) : ((28u << 8) | (16u << 16) | (255u << 24)));
      dv.pipe_pad = (e->pipe_timing ? 1u : 0u) | plan;
      if (e->h_dbg) memset(e->h_dbg, 0, 64 * 4);
      void* args[] = {(void*)&dv};
      const void* kfn = D.class_pref ? (const void*)cycle_kernel<3, 2, 1> : (const void*)cycle_kernel<3, 2, 0>;
      CUDA_TRY(e, cudaLaunchCooperativeKernel(kfn, dim3(D.pipe_S + 1), dim3(PIPE_THREADS), args, e->pipe_smem, e->stream));
      launches += 1;
    } else if (use_graph) {
      CUDA_TRY(e, cudaGraphLaunch(e->graph_exec, e->stream));
      launches += e->graph_launches;
    } else {
      uint32_t kernels = 0;
      if (const int rc = enqueue_links(e, D, backfill, false, batch, &kernels)) return rc;
      launches += kernels;
    }
    CUDA_TRY(e, cudaMemcpyAsync(e->h_ctl, D.ctl, sizeof(Ctl), cudaMemcpyDeviceToHost, e->stream));
    if (use_pipe && e->watchdog_s > 0) {
      // a persistent cooperative kernel that deadlocks cannot be cancelled from the host: poll instead of blocking, and if the
      // cycle is still running after watchdog_s say where it stands and abort the process (the driver then resets the context)
      const auto t0 = std::chrono::steady_clock::now();
      cudaError_t q;
      while ((q = cudaStreamQuery(e->stream)) == cudaErrorNotReady) {
        if (std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count() > e->watchdog_s) {
          fprintf(stderr, "libkbgpu: cycle_kernel did not finish within %.0f s — aborting.", e->watchdog_s);
          if (e->h_dbg) { fprintf(stderr, " progress words:"); for (int i = 0; i < 32; ++i) fprintf(stderr, " %u", e->h_dbg[i]); }
          fprintf(stderr, "\n");
          fflush(stderr);
          _exit(86);
        }
      }
      if (q != cudaSuccess) return fail(e, KB_E_CUDA, "cycle_kernel failed: %s", cudaGetErrorString(q));
    }
    CUDA_TRY(e, cudaStreamSynchronize(e->stream));
    if (e->h_ctl->done) break;
    if (use_pipe) return fail(e, e->h_ctl->error == 3 ? KB_E_CUDA : KB_E_STATE, "cycle_kernel ended without finishing the cycle (device error %u)", e->h_ctl->error);
    if (launches > cap) return fail(e, KB_E_STATE, "%s cycle did not terminate within %llu launches", backfill ? "backfill" : "allocate", (unsigned long long)cap);
  }
  e->last_launches = launches;
  if (in_cycle) {
    if (e->h_ctl->error == 2) return fail(e, KB_E_NCCL, "peer-memory exchange timed out waiting for another rank");
    if (e->h_ctl->error) return fail(e, KB_E_STATE, "device reported invariant violation %u", e->h_ctl->error);
    return KB_OK;
  }
  return finish_cycle(e, backfill, e->d_job_ready0, out, stats, launches, backfill ? 16u : BATCH, use_pipe);
}

// gang commit (K4), read-back of the decision table and the statistics of the view that ran last
int finish_cycle(kb_engine* e, const bool backfill, const int32_t* d_ready_start, kb_decision* out, kb_stats* stats, uint32_t launches,
                 const uint32_t batch, const bool use_pipe) {
  const DevSession& D = backfill ? e->dev_bf : e->dev;
  if (e->J) {
    const uint32_t warps_per_block = 4;
    gang_commit_kernel<<<(e->J + warps_per_block - 1) / warps_per_block, warps_per_block * 32, 0, e->stream>>>(
        e->dev, d_ready_start, e->dev_bf.ord_task, e->dev_bf.job_ord_off, e->dev_bf.job_pos);
    launches += 1;
  }
  CUDA_TRY(e, cudaGetLastError());
  if (e->T) CUDA_TRY(e, cudaMemcpyAsync(e->h_dec, e->dev.dec, (size_t)e->T * sizeof(kb_decision), cudaMemcpyDeviceToHost, e->stream));
  std::vector<uint32_t> placed(e->J);
  std::vector<int32_t> ready(e->J);
  if (e->J) {
    CUDA_TRY(e, cudaMemcpyAsync(placed.data(), e->dev.job_placed, (size_t)e->J * 4, cudaMemcpyDeviceToHost, e->stream));
    CUDA_TRY(e, cudaMemcpyAsync(ready.data(), e->dev.job_ready, (size_t)e->J * 4, cudaMemcpyDeviceToHost, e->stream));
  }
  CUDA_TRY(e, cudaEventRecord(e->ev1, e->stream));
  CUDA_TRY(e, cudaStreamSynchronize(e->stream));
  if (e->h_ctl->error == 2) return fail(e, KB_E_NCCL, "peer-memory exchange timed out waiting for another rank");
  if (e->h_ctl->error) return fail(e, KB_E_STATE, "device reported invariant violation %u", e->h_ctl->error);
  if (out && e->T) memcpy(out, e->h_dec, (size_t)e->T * sizeof(kb_decision));
  if (stats) {
    const Ctl& c = *e->h_ctl;
    memset(stats, 0, sizeof *stats);
    stats->pairs_logical = c.pairs_logical; stats->pairs_scanned = c.pairs_scanned; stats->pairs_replayed = c.pairs_replayed;
    stats->tasks_processed = c.tasks_processed; stats->tasks_allocated = c.tasks_allocated; stats->tasks_pipelined = c.tasks_pipelined;
    stats->visits = c.visits; stats->kernel_launches = launches; stats->n_classes = e->C;
    uint32_t jr = 0;
    for (uint32_t j = 0; j < e->J; ++j)
      if (placed[j] && (!e->gang_ready || ready[j] >= e->job_min_avail_host[j])) ++jr;
    stats->jobs_ready = jr;
    float ms = 0; cudaEventElapsedTime(&ms, e->ev0, e->ev1);
    stats->gpu_ms = ms; stats->load_ms = e->load_ms;
    stats->scans = c.scans; stats->rescans = c.rescans;
    stats->cyc_scan = c.cyc_scan; stats->cyc_merge = c.cyc_merge; stats->cyc_replay = c.cyc_replay; stats->cyc_total = c.cyc_total; stats->cyc_steps = c.cyc_steps; stats->cyc_ctl = c.cyc_ctl; stats->cyc_ring = c.cyc_ring; stats->cyc_plan = c.cyc_plan;
    stats->pipe_builds_used = c.pipe_builds_used; stats->pipe_builds_missed = c.pipe_builds_missed; stats->pipe_builds_cancelled = c.pipe_builds_cancelled;
    stats->predictions = c.predictions; stats->mispredictions = c.mispredictions;
    stats->chain_hits = c.chain_hits;
    stats->exchange_mode = e->world == 1 ? 0u : (e->replicated ? 3u : (D.p2p ? 2u : 1u));
    stats->pipe_requests = c.pipe_requests; stats->pipe_urgent = c.pipe_urgent; stats->pipe_extends = c.pipe_extends;
    stats->pipe_patched = c.pipe_patched; stats->pipe_patch_entries = c.pipe_patch_entries; stats->pipeline = use_pipe ? 1u : 0u;
    stats->h2d_bytes = backfill ? 0 : (uint64_t)e->mut_bytes + e->imm_bytes;
    stats->d2h_bytes = (uint64_t)e->T * sizeof(kb_decision) + (uint64_t)e->J * 8 + (uint64_t)(launches / batch) * sizeof(Ctl);
  }
  return KB_OK;
}

}  // namespace

int kb_allocate(kb_engine* e, kb_decision* out, kb_stats* stats) {
  if (!e) return KB_E_BADARG;
  if (!e->loaded) return fail(e, KB_E_STATE, "kb_allocate before kb_session_load");
  return run_action(e, false, out, stats);
}

int kb_backfill(kb_engine* e, kb_decision* out, kb_stats* stats) {
  if (!e) return KB_E_BADARG;
  if (!e->loaded) return fail(e, KB_E_STATE, "kb_backfill before kb_session_load");
  return run_action(e, true, out, stats);
}

int kb_session_load_running(kb_engine* e, const kb_snapshot* s, const kb_running* run) {
  if (!e) return KB_E_BADARG;
  if (!e->loaded) return fail(e, KB_E_STATE, "kb_session_load_running before kb_session_load");
  if (!s || s->N != e->N || s->T != e->T || s->J != e->J || s->Q != e->Q || s->R != e->R)
    return fail(e, KB_E_BADARG, "kb_session_load_running: `snap` is not the snapshot of the loaded session");
  if (e->world > 1 && !e->replicated) return fail(e, KB_E_UNSUPPORTED_FEATURE, "reclaim / preempt run on the full node table: not with KB_ENGINE_SHARD");
  // counter path: refused when a pending class reads a counter group in predicate step 10 (kb_build.h aff_groups_unread)
  if (e->built.aff_session && !e->built.aff_evict_ok)
    return fail(e, KB_E_UNSUPPORTED_FEATURE, "reclaim / preempt in this session with inter-pod affinity are outside this build: the victim walk does not "
                "update the affinity counters (only host-level anti-affinity, kept as bits of the node records, runs the evicting actions)");
  CUDA_TRY(e, cudaSetDevice(e->device));
  e->running_loaded = false;
  BuildErr be;
  DevSession H{};
  e->built.bind(H, e->built.mut.host.data(), e->built.imm.host.data());      // host view of the as-loaded state: the heaps' comparators read it
  const int rc = build_evict(s, run, e->built, H, e->ev_built, &be);
  if (rc) return fail(e, rc, "%s", be.msg.c_str());
  const size_t ib = e->ev_built.imm.host.size(), mb = e->ev_built.mut.host.size();
  if (ib > e->ev_cap_imm) {
    if (e->d_ev_imm) cudaFree(e->d_ev_imm);
    e->d_ev_imm = nullptr; e->ev_cap_imm = 0;
    CUDA_TRY(e, cudaMalloc(&e->d_ev_imm, ib + ib / 4));
    e->ev_cap_imm = ib + ib / 4;
  }
  if (mb > e->ev_cap_mut) {
    if (e->d_ev_mut) cudaFree(e->d_ev_mut);
    if (e->d_ev_pristine) cudaFree(e->d_ev_pristine);
    e->d_ev_mut = e->d_ev_pristine = nullptr; e->ev_cap_mut = 0;
    CUDA_TRY(e, cudaMalloc(&e->d_ev_mut, mb + mb / 4));
    CUDA_TRY(e, cudaMalloc(&e->d_ev_pristine, mb + mb / 4));
    e->ev_cap_mut = mb + mb / 4;
  }
  CUDA_TRY(e, cudaMemcpyAsync(e->d_ev_imm, e->ev_built.imm.host.data(), ib, cudaMemcpyHostToDevice, e->stream));
  CUDA_TRY(e, cudaMemcpyAsync(e->d_ev_pristine, e->ev_built.mut.host.data(), mb, cudaMemcpyHostToDevice, e->stream));
  CUDA_TRY(e, cudaStreamSynchronize(e->stream));
  e->ev_built.bind(e->ev, e->d_ev_imm, e->d_ev_mut);
  e->running_loaded = true;
  return KB_OK;
}

namespace {
__global__ void carry_u32_kernel(const uint32_t* __restrict__ src, uint32_t* __restrict__ dst) { if (threadIdx.x == 0 && blockIdx.x == 0) *dst = *src; }
__global__ void prep_allocate_kernel(const __grid_constant__ DevSession S, const uint32_t* __restrict__ step_src) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  prep_task_lists(S);
  prep_allocate(S, *S.ctl, step_src ? *step_src : 0u);
}
__global__ void prep_backfill_kernel(const __grid_constant__ DevSession Sbf, const uint32_t* __restrict__ step_src) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  prep_backfill(Sbf, *Sbf.ctl, step_src ? *step_src : 0u);
}
}  // namespace

// scheduler.go:88-101 on the device: the action list on ONE session
int kb_cycle(kb_engine* e, const uint8_t* actions, uint32_t n_actions, kb_decision* out, uint8_t* evicted, uint32_t* evict_order,
             uint32_t* bounds, kb_stats* stats) {
  if (!e) return KB_E_BADARG;
  if (!e->loaded) return fail(e, KB_E_STATE, "kb_cycle before kb_session_load");
  if (!actions && n_actions) return fail(e, KB_E_BADARG, "actions is NULL");
  uint32_t n_alloc = 0, n_bf = 0;
  for (uint32_t i = 0; i < n_actions; ++i) {
    if (actions[i] > KB_ACT_PREEMPT) return fail(e, KB_E_BADARG, "unknown action %u", actions[i]);
    n_alloc += actions[i] == KB_ACT_ALLOCATE; n_bf += actions[i] == KB_ACT_BACKFILL;
    if ((actions[i] == KB_ACT_RECLAIM || actions[i] == KB_ACT_PREEMPT) && !e->running_loaded)
      return fail(e, KB_E_STATE, "%s before kb_session_load_running", actions[i] == KB_ACT_RECLAIM ? "reclaim" : "preempt");
  }
  if (n_alloc > 1 || n_bf > 1) return fail(e, KB_E_BADARG, "at most one allocate and one backfill per cycle");
  // A discarded Statement leaves TaskInfo.NodeName of its un-pipelined tasks behind (statement.go:153-188 never clears it), and
  // the next ssn.Allocate / ssn.Pipeline of such a task on another node fails in NodeInfo.AddTask AFTER the status changed
  // (node_info.go:173-176, session.go:241-262).  The shipped action order runs preempt last; other orders are refused
  // rather than modelled.
  for (uint32_t i = 0; i + 1 < n_actions; ++i)
    if (actions[i] == KB_ACT_PREEMPT && actions[i + 1] != KB_ACT_PREEMPT)
      return fail(e, KB_E_UNSUPPORTED_FEATURE, "an action after preempt: a discarded Statement leaves TaskInfo.NodeName behind (statement.go:153-188), outside this build");
  CUDA_TRY(e, cudaSetDevice(e->device));
  CUDA_TRY(e, cudaEventRecord(e->ev0, e->stream));
  CUDA_TRY(e, restore_session(e));
  e->allocate_ran = false;
  if ((size_t)e->J * 4 > e->cap_ready_start) {
    if (e->d_ready_start) cudaFree(e->d_ready_start);
  if (e->d_bind_scratch) cudaFree(e->d_bind_scratch);
  e->d_bind_scratch = nullptr; e->cap_bind_scratch = 0;
    e->d_ready_start = nullptr; e->cap_ready_start = 0;
    CUDA_TRY(e, cudaMalloc(&e->d_ready_start, (size_t)std::max(1u, e->J) * 4));
    e->cap_ready_start = (size_t)std::max(1u, e->J) * 4;
  }
  const uint32_t* step_alloc = (const uint32_t*)((const char*)e->dev.ctl + offsetof(Ctl, step));
  const uint32_t* step_bf = (const uint32_t*)((const char*)e->dev_bf.ctl + offsetof(Ctl, step));
  uint32_t* step_ev = e->running_loaded ? (uint32_t*)((char*)e->ev.ctl + offsetof(EvictCtl, step)) : nullptr;
  const uint32_t* nev_ev = e->running_loaded ? (const uint32_t*)((const char*)e->ev.ctl + offsetof(EvictCtl, n_evicted)) : nullptr;
  const uint32_t* latest = nullptr;          // who holds the session's step counter
  bool dirty = false;                        // an earlier action of this cycle changed what allocate / backfill set up at load
  bool ready_taken = false, bf_last = false, placed_ran = false;
  uint32_t launches = 0;
  bool use_pipe = false;
  std::vector<uint32_t> hb(2 * (size_t)std::max(1u, n_actions), 0);
  uint32_t* d_bounds = nullptr;
  CUDA_TRY(e, cudaMalloc(&d_bounds, hb.size() * 4));
  CUDA_TRY(e, cudaMemsetAsync(d_bounds, 0, hb.size() * 4, e->stream));
  struct Free { uint32_t* p; ~Free() { if (p) cudaFree(p); } } free_bounds{d_bounds};
  bool session_dead = false;                 // Ctl.pred_dead after a backfill: every later ssn.PredicateFn of the session fails
  for (uint32_t i = 0; i < n_actions; ++i) {
    const uint8_t a = actions[i];
    if (session_dead) {                      // the remaining actions find no node for anybody: nothing to launch
      if (latest) carry_u32_kernel<<<1, 1, 0, e->stream>>>(latest, d_bounds + 2 * i);
      if (nev_ev) carry_u32_kernel<<<1, 1, 0, e->stream>>>(nev_ev, d_bounds + 2 * i + 1);
      continue;
    }
    if (a == KB_ACT_RECLAIM || a == KB_ACT_PREEMPT) {
      if (latest && latest != step_ev) carry_u32_kernel<<<1, 1, 0, e->stream>>>(latest, step_ev);
      CUDA_TRY(e, launch_evict(a == KB_ACT_PREEMPT, e->dev, e->ev, e->coop_ok ? e->sm_count : 1, e->stream));
      launches += 1;
      latest = step_ev; dirty = true;
    } else {
      const bool bf = a == KB_ACT_BACKFILL;
      if (!ready_taken) {            // ssn.JobReady inside ssn.Allocate counts from the ReadyTaskNum the placing actions found
        CUDA_TRY(e, cudaMemcpyAsync(e->d_ready_start, e->dev.job_ready, (size_t)e->J * 4, cudaMemcpyDeviceToDevice, e->stream));
        ready_taken = true;
      }
      if (!bf) {
        if (dirty || latest) { prep_allocate_kernel<<<1, 1, 0, e->stream>>>(e->dev, latest); e->imm_dirty = true; }
        use_pipe = e->dev.pipe != 0;
      } else {
        if (dirty) { prep_backfill_kernel<<<1, 1, 0, e->stream>>>(e->dev_bf, latest); e->imm_dirty = true; }
        else seed_backfill_kernel<<<1, 32, 0, e->stream>>>(e->dev.ctl, e->dev_bf.ctl, e->allocate_ran ? 1 : 0);
      }
      CUDA_TRY(e, cudaGetLastError());
      const int rc = run_action(e, bf, nullptr, nullptr, true);
      if (rc) return rc;
      launches += e->last_launches;
      if (bf && e->h_ctl->pred_dead) session_dead = true;
      latest = bf ? step_bf : step_alloc;
      bf_last = bf; placed_ran = true;
      // a later evicting action must see the placements: they are in the decision table and the node / job tables already
      dirty = dirty || false;
    }
    if (latest) carry_u32_kernel<<<1, 1, 0, e->stream>>>(latest, d_bounds + 2 * i);
    if (nev_ev) carry_u32_kernel<<<1, 1, 0, e->stream>>>(nev_ev, d_bounds + 2 * i + 1);
  }
  CUDA_TRY(e, cudaMemcpyAsync(hb.data(), d_bounds, hb.size() * 4, cudaMemcpyDeviceToHost, e->stream));
  // evictions
  const uint32_t n = e->running_loaded ? e->ev_built.n_run : 0;
  std::vector<uint32_t> order(std::max(1u, n));
  EvictCtl ectl{};
  if (n) CUDA_TRY(e, cudaMemcpyAsync(order.data(), e->ev.evict_order, (size_t)n * 4, cudaMemcpyDeviceToHost, e->stream));
  if (e->running_loaded) CUDA_TRY(e, cudaMemcpyAsync(&ectl, e->ev.ctl, sizeof ectl, cudaMemcpyDeviceToHost, e->stream));
  if (!placed_ran) {
    // no placing action ran: the control block the statistics come from is the allocate view's as loaded
    CUDA_TRY(e, cudaMemcpyAsync(e->h_ctl, e->dev.ctl, sizeof(Ctl), cudaMemcpyDeviceToHost, e->stream));
  }
  int rc = finish_cycle(e, bf_last, ready_taken ? e->d_ready_start : e->d_job_ready0, out, stats, launches, BATCH, use_pipe);
  if (rc) return rc;
  if (ectl.error == 2) return fail(e, KB_E_UNSUPPORTED_FEATURE, "a node hands more than %u victims to one preemptor", KB_EVICT_MAXV);
  if (ectl.error == 3) return fail(e, KB_E_UNSUPPORTED_FEATURE, "a member of an inter-pod affinity counter group was evicted (KB_RUNNING_AFF_MEMBER): the member bits "
                                   "of the node records are stale from that point on, the outcome of this cycle is withheld");
  if (ectl.error) return fail(e, KB_E_STATE, "the reference would panic here: Resource.Sub on an insufficient resource (resource_info.go:158)");
  if (n) {
    const uint32_t* r_orig = (const uint32_t*)(e->ev_built.imm.host.data() + e->ev_built.oi.r_orig);
    for (uint32_t k = 0; k < n; ++k) {
      const uint32_t i = r_orig[k];
      if (evicted) evicted[i] = order[k] != 0xFFFFFFFFu ? 1 : 0;
      if (evict_order) evict_order[i] = order[k];
    }
  }
  if (bounds) for (uint32_t i = 0; i < 2 * n_actions; ++i) bounds[i] = hb[i];
  if (stats) {
    if (!placed_ran) { stats->pairs_logical = 0; stats->pairs_scanned = 0; stats->tasks_processed = 0; stats->tasks_pipelined = 0; }
    stats->pairs_logical += ectl.pairs_logical; stats->pairs_scanned += (uint64_t)ectl.scans * e->N;
    stats->tasks_processed += ectl.tasks_processed; stats->tasks_pipelined += ectl.n_pipelined;
    stats->evictions = ectl.n_evicted; stats->evict_sweeps = ectl.scans;
    stats->d2h_bytes += (uint64_t)n * 4 + sizeof ectl;
  }
  return KB_OK;
}

int kb_reclaim(kb_engine* e, kb_decision* out, uint8_t* evicted, uint32_t* evict_order, kb_stats* stats) {
  const uint8_t a = KB_ACT_RECLAIM;
  return kb_cycle(e, &a, 1, out, evicted, evict_order, nullptr, stats);
}

int kb_preempt(kb_engine* e, kb_decision* out, uint8_t* evicted, uint32_t* evict_order, kb_stats* stats) {
  const uint8_t a = KB_ACT_PREEMPT;
  return kb_cycle(e, &a, 1, out, evicted, evict_order, nullptr, stats);
}

int kb_bind_list(kb_engine* e, uint32_t* task, int32_t* node, uint32_t* n) {
  if (!e || !n) return KB_E_BADARG;
  if (!e->loaded) return fail(e, KB_E_STATE, "kb_bind_list before kb_session_load");
  *n = 0;
  if (e->T == 0) return KB_OK;
  if (!task || !node) return fail(e, KB_E_BADARG, "kb_bind_list: NULL output");
  CUDA_TRY(e, cudaSetDevice(e->device));
  const size_t need = bind_scratch_bytes(e->T);
  if (need > e->cap_bind_scratch) {
    if (e->d_bind_scratch) cudaFree(e->d_bind_scratch);
    e->d_bind_scratch = nullptr; e->cap_bind_scratch = 0;
    CUDA_TRY(e, cudaMalloc(&e->d_bind_scratch, need + need / 4));
    e->cap_bind_scratch = need + need / 4;
  }
  cudaEventRecord(e->ev0, e->stream);
  const cudaError_t c = bind_list(e->dev.dec, e->T, e->d_bind_scratch, e->cap_bind_scratch, task, node, n, e->stream);
  cudaEventRecord(e->ev1, e->stream);
  if (c != cudaSuccess) return fail(e, KB_E_CUDA, "kb_bind_list: %s", cudaGetErrorString(c));
  cudaEventSynchronize(e->ev1);
  cudaEventElapsedTime(&e->last_kernel_ms, e->ev0, e->ev1);
  return KB_OK;
}

int kb_predicate_score(kb_engine* e, uint32_t task_lo, uint32_t task_hi, uint8_t* fit, double* score) {
  if (!e) return KB_E_BADARG;
  if (!e->loaded) return fail(e, KB_E_STATE, "kb_predicate_score before kb_session_load");
  if (e->built.aff.on && score && (e->built.aff.has_weights || e->built.aff.has_pref))
    return fail(e, KB_E_UNSUPPORTED_FEATURE, "kb_predicate_score: InterPodAffinityPriority / NodeAffinityPriority need reductions over the feasible nodes; "
                "ask for `fit` only (predicate step 10 is evaluated against the current counters)");
  if (task_lo > task_hi || task_hi > e->T) return fail(e, KB_E_BADARG, "task range [%u,%u) outside [0,%u)", task_lo, task_hi, e->T);
  const size_t n = (size_t)(task_hi - task_lo) * e->N;
  if (n == 0 || e->NT == 0) return KB_OK;
  CUDA_TRY(e, cudaSetDevice(e->device));
  uint8_t* d_fit = nullptr; double* d_score = nullptr;
  if (fit) CUDA_TRY(e, cudaMalloc(&d_fit, n));
  if (score) {
    const cudaError_t ca = cudaMalloc(&d_score, n * 8);
    if (ca != cudaSuccess) { if (d_fit) cudaFree(d_fit); return fail(e, KB_E_CUDA, "cudaMalloc(score) failed: %s", cudaGetErrorString(ca)); }   // no leak of d_fit
  }
  dim3 grid(e->NT, (task_hi - task_lo + MATRIX_TASKS_PER_CTA - 1) / MATRIX_TASKS_PER_CTA);
  cudaEventRecord(e->ev0, e->stream);
  with_rec(e->built.rec, [&](auto t) {
    matrix_kernel<typename decltype(t)::type><<<grid, MATRIX_THREADS, e->tile_smem, e->stream>>>(e->dev, e->d_task_class, task_lo, task_hi, d_fit, d_score);
  });
  cudaEventRecord(e->ev1, e->stream);
  cudaError_t c = cudaGetLastError();
  if (c == cudaSuccess && fit) c = cudaMemcpyAsync(fit, d_fit, n, cudaMemcpyDeviceToHost, e->stream);
  if (c == cudaSuccess && score) c = cudaMemcpyAsync(score, d_score, n * 8, cudaMemcpyDeviceToHost, e->stream);
  if (c == cudaSuccess) c = cudaStreamSynchronize(e->stream);
  if (d_fit) cudaFree(d_fit);
  if (d_score) cudaFree(d_score);
  if (c != cudaSuccess) return fail(e, KB_E_CUDA, "matrix_kernel: %s", cudaGetErrorString(c));
  cudaEventElapsedTime(&e->last_kernel_ms, e->ev0, e->ev1);
  return KB_OK;
}

int kb_best_nodes(kb_engine* e, uint32_t task_lo, uint32_t task_hi, uint64_t* best_key) {
  if (!e) return KB_E_BADARG;
  if (!e->loaded) return fail(e, KB_E_STATE, "kb_best_nodes before kb_session_load");
  if (e->built.aff.on) return fail(e, KB_E_UNSUPPORTED_FEATURE, "kb_best_nodes: the matrix kernels do not evaluate inter-pod affinity");
  if (task_lo > task_hi || task_hi > e->T || !best_key) return fail(e, KB_E_BADARG, "bad task range or NULL output");
  const uint32_t n = task_hi - task_lo;
  if (n == 0) return KB_OK;
  CUDA_TRY(e, cudaSetDevice(e->device));
  unsigned long long* d_best = nullptr;
  CUDA_TRY(e, cudaMalloc(&d_best, (size_t)n * 8));
  cudaError_t c = cudaMemsetAsync(d_best, 0, (size_t)n * 8, e->stream);
  if (c == cudaSuccess && e->NT) {
    // enough task chunks to fill the machine a few times over, each CTA keeps its node tile in shared memory
    uint32_t chunks = std::max(1u, std::min(n, (uint32_t)(8 * e->sm_count + e->NT - 1) / std::max(1u, e->NT)));
    dim3 grid(e->NT, chunks);
    cudaEventRecord(e->ev0, e->stream);
    with_rec(e->built.rec, [&](auto t) {
      best_nodes_kernel<typename decltype(t)::type><<<grid, MATRIX_THREADS, e->tile_smem, e->stream>>>(e->dev, e->d_task_class, task_lo, task_hi, d_best);
    });
    cudaEventRecord(e->ev1, e->stream);
    c = cudaGetLastError();
  }
  if (c == cudaSuccess) c = cudaMemcpyAsync(best_key, d_best, (size_t)n * 8, cudaMemcpyDeviceToHost, e->stream);
  if (c == cudaSuccess) c = cudaStreamSynchronize(e->stream);
  cudaFree(d_best);
  if (c != cudaSuccess) return fail(e, KB_E_CUDA, "best_nodes_kernel: %s", cudaGetErrorString(c));
  cudaEventElapsedTime(&e->last_kernel_ms, e->ev0, e->ev1);
  return KB_OK;
}

int kb_last_kernel_ms(kb_engine* e, float* ms) {
  if (!e || !ms) return KB_E_BADARG;
  *ms = e->last_kernel_ms;
  return KB_OK;
}

int kb_node_state(kb_engine* e, double* idle, double* releasing, double* used, int32_t* pods, int64_t* nz_cpu, int64_t* nz_mem, uint64_t* ports) {
  if (!e) return KB_E_BADARG;
  if (!e->loaded) return fail(e, KB_E_STATE, "kb_node_state before kb_session_load");
  CUDA_TRY(e, cudaSetDevice(e->device));
  const uint32_t R = e->R, W = e->W, N = e->N;
  const size_t tile_u64 = (size_t)e->ncols * TILE_NODES;
  std::vector<uint64_t> tiles((size_t)std::max(1u, e->NT) * tile_u64);
  std::vector<double> usedv((size_t)R * std::max(1u, N));
  CUDA_TRY(e, cudaMemcpyAsync(tiles.data(), e->dev.tiles, (size_t)e->NT * tile_u64 * 8, cudaMemcpyDeviceToHost, e->stream));
  CUDA_TRY(e, cudaMemcpyAsync(usedv.data(), e->dev.node_used, (size_t)R * N * 8, cudaMemcpyDeviceToHost, e->stream));
  CUDA_TRY(e, cudaStreamSynchronize(e->stream));
  for (uint32_t n = 0; n < N; ++n) {
    TileAcc a{tiles.data() + (size_t)(n / TILE_NODES) * tile_u64, n % TILE_NODES, R, W};
    for (uint32_t r = 0; r < R; ++r) {
      if (idle) idle[(size_t)r * N + n] = a.idle(r);
      if (releasing) releasing[(size_t)r * N + n] = a.rel(r);
      if (used) used[(size_t)r * N + n] = usedv[(size_t)r * N + n];
    }
    if (pods) pods[n] = a.pods();
    if (nz_cpu) nz_cpu[n] = a.nz_cpu();
    if (nz_mem) nz_mem[n] = a.nz_mem();
    if (ports) for (uint32_t w = 0; w < W; ++w) ports[(size_t)w * N + n] = a.ports(w) & ~e->built.aff_atom_mask[w];      // host-level anti-affinity bits are not ports
  }
  return KB_OK;
}

int kb_order_state(kb_engine* e, double* job_share, int32_t* job_ready, double* queue_share, double* queue_deserved, double* queue_allocated) {
  if (!e) return KB_E_BADARG;
  if (!e->loaded) return fail(e, KB_E_STATE, "kb_order_state before kb_session_load");
  CUDA_TRY(e, cudaSetDevice(e->device));
  if (job_share && e->J) CUDA_TRY(e, cudaMemcpyAsync(job_share, e->dev.job_share, (size_t)e->J * 8, cudaMemcpyDeviceToHost, e->stream));
  if (job_ready && e->J) CUDA_TRY(e, cudaMemcpyAsync(job_ready, e->dev.job_ready, (size_t)e->J * 4, cudaMemcpyDeviceToHost, e->stream));
  if (queue_share && e->Q) CUDA_TRY(e, cudaMemcpyAsync(queue_share, e->dev.q_share, (size_t)e->Q * 8, cudaMemcpyDeviceToHost, e->stream));
  if (queue_deserved && e->Q) CUDA_TRY(e, cudaMemcpyAsync(queue_deserved, e->dev.q_deserved, (size_t)e->R * e->Q * 8, cudaMemcpyDeviceToHost, e->stream));
  if (queue_allocated && e->Q) CUDA_TRY(e, cudaMemcpyAsync(queue_allocated, e->dev.q_allocated, (size_t)e->R * e->Q * 8, cudaMemcpyDeviceToHost, e->stream));
  CUDA_TRY(e, cudaStreamSynchronize(e->stream));
  return KB_OK;
}

}  // extern "C"
