// core_probe.cu — both builds of the engine's shared arithmetic (kb_core.h, kb_aff.h) behind one C entry point per function,
// so that tests/test_core_arith.py (host) and tests/test_gpu_core_arith.py (device) check them against one Python reference.
//
// Every entry point takes host arrays of n cases.  device = 0 runs the KB_HD function on the host, in this process, without a
// single CUDA runtime call (the CPU tests load the library on machines without a GPU); device = 1 copies the arrays to the GPU,
// runs one kernel over them, and copies the results back.  Returns 0, or the cudaError_t of the first failing call.
// Nothing here restates the production functions: the per-case bodies below only call them.
#include <cuda_runtime.h>

#include <stddef.h>
#include <stdint.h>

#include "../../kube_batch_b200/csrc/kb_ctl.h"     // TileAcc (+ kb_core.h, kb_aff.h)

namespace {

constexpr int MAX_BUFS = 8;
struct Bufs { void* p[MAX_BUFS]; };
struct Arg { void* host; size_t bytes; bool out; };

template <class Op>
__global__ void probe_kernel(Bufs b, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) Op::apply(b, i);
}

template <class Op>
int run(int device, size_t n, const Arg* args, int nargs) {
  Bufs hb{}, db{};
  for (int k = 0; k < nargs; ++k) hb.p[k] = args[k].host;
  if (!device) {
    for (size_t i = 0; i < n; ++i) Op::apply(hb, i);
    return 0;
  }
  cudaError_t e = cudaSuccess;
  int made = 0;
  for (; made < nargs && e == cudaSuccess; ++made) {
    e = cudaMalloc(&db.p[made], args[made].bytes ? args[made].bytes : 8);
    if (e == cudaSuccess && args[made].bytes) e = cudaMemcpy(db.p[made], args[made].host, args[made].bytes, cudaMemcpyHostToDevice);
  }
  if (e == cudaSuccess && n) {
    const unsigned blocks = (unsigned)((n + 255) / 256 < 4096 ? (n + 255) / 256 : 4096);
    probe_kernel<Op><<<blocks, 256>>>(db, n);
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
  }
  for (int k = 0; k < nargs && e == cudaSuccess; ++k)
    if (args[k].out && args[k].bytes) e = cudaMemcpy(args[k].host, db.p[k], args[k].bytes, cudaMemcpyDeviceToHost);
  for (int k = 0; k < made; ++k) cudaFree(db.p[k]);
  return (int)e;
}

#define I64(k) ((int64_t*)b.p[k])
#define U64(k) ((uint64_t*)b.p[k])
#define F64(k) ((double*)b.p[k])
#define U8(k) ((uint8_t*)b.p[k])

struct DivOp { static KB_HD void apply(const Bufs& b, size_t i) { I64(2)[i] = kb::div_0_to_10(I64(0)[i], I64(1)[i]); } };
struct LeastOp { static KB_HD void apply(const Bufs& b, size_t i) { I64(2)[i] = kb::least_requested_score(I64(0)[i], I64(1)[i]); } };
struct MostOp { static KB_HD void apply(const Bufs& b, size_t i) { I64(2)[i] = kb::most_requested_score(I64(0)[i], I64(1)[i]); } };
struct BalancedOp {
  static KB_HD void apply(const Bufs& b, size_t i) { I64(4)[i] = kb::balanced_score(I64(0)[i], I64(1)[i], I64(2)[i], I64(3)[i]); }
};
struct LeOp { static KB_HD void apply(const Bufs& b, size_t i) { U8(3)[i] = kb::le_func(F64(0)[i], F64(1)[i], F64(2)[i]) ? 1 : 0; } };
// p[3] holds R
struct ResLeOp {
  static KB_HD void apply(const Bufs& b, size_t i) {
    const uint32_t R = (uint32_t)I64(3)[0];
    const double* l = F64(0) + i * R;
    const double* r = F64(1) + i * R;
    U8(2)[i] = kb::res_less_equal(R, [&](uint32_t k) { return l[k]; }, [&](uint32_t k) { return r[k]; }) ? 1 : 0;
  }
};
struct AffScoreOp { static KB_HD void apply(const Bufs& b, size_t i) { I64(3)[i] = kb::aff_score(I64(0)[i], I64(1)[i], I64(2)[i]); } };
struct AddPrefOp {
  static KB_HD void apply(const Bufs& b, size_t i) { U64(4)[i] = kb::add_pref_term(U64(0)[i], I64(1)[i], I64(2)[i], I64(3)[i]); }
};
struct AffAddOp {
  static KB_HD void apply(const Bufs& b, size_t i) { U64(3)[i] = kb::aff_add_score(U64(0)[i], (int32_t)I64(1)[i], I64(2)[i]); }
};
// pair i: class cls[i] on node i of the packed tiles ([tile][ncols][TILE_NODES], the node table's layout)
template <int RR, int WW>
struct EvalOp {
  static KB_HD void apply(const Bufs& b, size_t i) {
    const kb::EvalConf& cf = *(const kb::EvalConf*)b.p[0];
    const kb::ClassRec& c = ((const kb::ClassRec*)b.p[1])[i];
    const uint32_t ncols = kb::tile_ncols(cf.R, cf.W);
    const kb::TileAcc acc{U64(2) + (i / kb::TILE_NODES) * (size_t)ncols * kb::TILE_NODES, (uint32_t)(i % kb::TILE_NODES), cf.R, cf.W};
    bool fi = false, pok = false;
    U64(3)[i] = kb::eval_pair<RR, WW>(cf, c, acc, (uint32_t)i, &fi, &pok);
    U8(4)[i] = fi ? 1 : 0;
    U8(5)[i] = pok ? 1 : 0;
  }
};

}  // namespace

extern "C" {

int kbp_sizeof_class_rec() { return (int)sizeof(kb::ClassRec); }
int kbp_sizeof_eval_conf() { return (int)sizeof(kb::EvalConf); }
int kbp_tile_nodes() { return kb::TILE_NODES; }

int kbp_div_0_to_10(int device, size_t n, int64_t* a, int64_t* b, int64_t* out) {
  const Arg args[] = {{a, n * 8, false}, {b, n * 8, false}, {out, n * 8, true}};
  return run<DivOp>(device, n, args, 3);
}
int kbp_least_requested(int device, size_t n, int64_t* req, int64_t* cap, int64_t* out) {
  const Arg args[] = {{req, n * 8, false}, {cap, n * 8, false}, {out, n * 8, true}};
  return run<LeastOp>(device, n, args, 3);
}
int kbp_most_requested(int device, size_t n, int64_t* req, int64_t* cap, int64_t* out) {
  const Arg args[] = {{req, n * 8, false}, {cap, n * 8, false}, {out, n * 8, true}};
  return run<MostOp>(device, n, args, 3);
}
int kbp_balanced(int device, size_t n, int64_t* rc, int64_t* cc, int64_t* rm, int64_t* cm, int64_t* out) {
  const Arg args[] = {{rc, n * 8, false}, {cc, n * 8, false}, {rm, n * 8, false}, {cm, n * 8, false}, {out, n * 8, true}};
  return run<BalancedOp>(device, n, args, 5);
}
int kbp_le_func(int device, size_t n, double* l, double* r, double* diff, uint8_t* out) {
  const Arg args[] = {{l, n * 8, false}, {r, n * 8, false}, {diff, n * 8, false}, {out, n, true}};
  return run<LeOp>(device, n, args, 4);
}
int kbp_res_less_equal(int device, size_t n, int64_t R, double* l, double* r, uint8_t* out) {
  int64_t rr = R;
  const Arg args[] = {{l, n * R * 8, false}, {r, n * R * 8, false}, {out, n, true}, {&rr, 8, false}};
  return run<ResLeOp>(device, n, args, 4);
}
int kbp_aff_score(int device, size_t n, int64_t* count, int64_t* mn, int64_t* mx, int64_t* out) {
  const Arg args[] = {{count, n * 8, false}, {mn, n * 8, false}, {mx, n * 8, false}, {out, n * 8, true}};
  return run<AffScoreOp>(device, n, args, 4);
}
int kbp_add_pref_term(int device, size_t n, uint64_t* key, int64_t* w, int64_t* count, int64_t* max_count, uint64_t* out) {
  const Arg args[] = {{key, n * 8, false}, {w, n * 8, false}, {count, n * 8, false}, {max_count, n * 8, false}, {out, n * 8, true}};
  return run<AddPrefOp>(device, n, args, 5);
}
int kbp_aff_add_score(int device, size_t n, uint64_t* key, int64_t* w_podaff, int64_t* score, uint64_t* out) {
  const Arg args[] = {{key, n * 8, false}, {w_podaff, n * 8, false}, {score, n * 8, false}, {out, n * 8, true}};
  return run<AffAddOp>(device, n, args, 4);
}
// geometry 1: eval_pair<3, 2> (the conf must say R = 3, W = 2); geometry 0: eval_pair<0, 0> (R, W read from the conf)
int kbp_eval_pair(int device, int geometry, size_t n, const void* conf, const void* cls, const uint64_t* tiles, uint64_t* key,
                  uint8_t* fits_idle, uint8_t* pred_ok) {
  const kb::EvalConf& cf = *(const kb::EvalConf*)conf;
  const size_t tiles_u64 = (n + kb::TILE_NODES - 1) / kb::TILE_NODES * (size_t)kb::tile_ncols(cf.R, cf.W) * kb::TILE_NODES;
  const Arg args[] = {{(void*)conf, sizeof(kb::EvalConf), false}, {(void*)cls, n * sizeof(kb::ClassRec), false},
                      {(void*)tiles, tiles_u64 * 8, false}, {key, n * 8, true}, {fits_idle, n, true}, {pred_ok, n, true}};
  if (geometry == 1) {
    if (cf.R != 3 || cf.W != 2) return -1;
    return run<EvalOp<3, 2>>(device, n, args, 6);
  }
  return run<EvalOp<0, 0>>(device, n, args, 6);
}

}  // extern "C"
