// Host-side state behind the opaque C handles.
#pragma once
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdio>
#include <string>
#include <vector>

#include "posediff_b200.h"

namespace pdb {

struct DenoiserWeights;  // denoiser.cuh
struct VitWeights;       // api_vit.cu

// cudaFuncSetAttribute is per device, not per context: the dynamic shared memory already requested for each kernel, kept once
// per device so that every context on it sees what the others asked for (a second context must not lower a size a first one
// launches with).
struct KernelAttrs {
  size_t ggs[16] = {}, den[16] = {}, att = 0;
  size_t ggs_repro[2] = {0, 0};  // the reproducible GGS instantiation, plain / paired layout
  bool tc = false, tc128 = false, tc_deep = false;
  bool tc_swap[3] = {false, false, false};  // swap-AB instantiations (32 / 64 / 96 tokens on the N side)
  size_t vit_att[2] = {0, 0};  // the forward attention kernel's copy in api_vit.cu / api_vit_train.cu
  size_t vit_att_bwd = 0;      // backbone attention backward (csrc/api_vit_train.cu)
  bool train_att = false;      // denoiser training attention, forward and backward (csrc/api_train.cu)
};

// device < device_count (the process's cudaGetDeviceCount)
inline KernelAttrs* kernel_attrs(int device, int device_count) {
  static std::vector<KernelAttrs> per_device((size_t)device_count);
  return &per_device[(size_t)device];
}

struct Context {
  int device = -1;
  int sm_count = 0;
  int cc_major = 0, cc_minor = 0;
  size_t smem_optin = 0;
  std::string error;
  long long launches = 0;
  // GGS workspace (grown on demand)
  void* ggs_ws = nullptr;
  size_t ggs_ws_bytes = 0;
  // denoiser
  DenoiserWeights* weights = nullptr;
  void* den_ws = nullptr;
  size_t den_ws_bytes = 0;
  // stage hand-over of the persistent denoiser kernel: 0 = group barriers (default), 1 = flag-carrying activation words, no
  // barriers (pdb_debug_denoiser_handover / PDB_DEN_FLAG; parity-identical but slower: every CTA polling an 80 KB tile
  // loads L2)
  int den_flag = 0;
  void* den_flag_ws = nullptr;
  size_t den_flag_ws_bytes = 0;
  unsigned den_tag = 1;  // next unused version tag (0 = never written)
  // per-timestep tables of the current DDIM prefix (pdb_sample_loop_ddim): sched [100][8], then tproj [100][512], indexed by
  // virtual timestep.  Allocated once, so its address never changes; rewritten, stream-ordered, before each loop.
  void* step_tab = nullptr;
  // stage timing probe of the GGS kernel (debug): [ctas][8] cycle sums
  long long* ggs_clock = nullptr;
  int ggs_clock_ctas = 0;
  bool den_clock = false;  // the probe buffer is handed to the denoiser kernel instead of the GGS kernel
  // tensor-core engine: one captured CUDA graph of a whole diffusion step, replayed once per step (t lives on the device)
  cudaGraphExec_t tc_graph = nullptr;
  std::vector<size_t> tc_graph_key;
  cudaStream_t tc_capture_stream = nullptr;
  cudaStream_t pack_stream = nullptr;  // match uploads of pdb_sample_loop_host_matches (overlap the unguided prefix)
  int tc_graph_nodes = 0;
  KernelAttrs* attr = nullptr;  // kernel_attrs(device)
  bool tc_pdl = true;  // programmatic dependent launch between the kernels of the tensor-core engine's step graph (PDB_TC_PDL=0: off)
  bool tc_swap = false;     // swap-AB tensor-core tiles for <= 96 tokens (pdb_debug_tc_swap); default off
  // image feature extractor (csrc/api_vit.cu)
  VitWeights* vit = nullptr;
  void* vit_ws = nullptr;
  size_t vit_ws_bytes = 0;
  int ggs_layout = 1;       // stream layout of match sets packed on this context (ggs_layout.cuh): 0 plain, 1 paired (default)
  int denoiser_engine = 0;  // 0 auto, 1 fp32 persistent kernel, 2 wgmma/TMA tiles (TF32)
  // pdb_set_reproducible: the same bits on every call (GGS with fixed-order sums and the slot exchange, tensor-core GEMMs without
  // split-K); read when work is enqueued
  bool reproducible = false;
  // optional per-kernel timing (bench.py roofline): event pairs per launch, kind 0 = GGS, 1 = denoiser
  bool profiling = false;
  struct Timed { cudaEvent_t a, b; int kind; };
  std::vector<Timed> timed;
  // match ingestion: pinned host staging + a small pool of device buffers (cudaFree is slow and synchronising)
  void* pin = nullptr;
  size_t pin_bytes = 0;
  std::vector<std::pair<void*, size_t>> pool;
  // staging for the host-buffer entry point
  void* stage = nullptr;
  size_t stage_bytes = 0;
  // image preprocessing (csrc/api_pre.cu): two pinned staging slots, the event of each slot's last upload, and the device copy
  // of every frame's touched rows
  void* pre_pin[2] = {nullptr, nullptr};
  size_t pre_pin_bytes[2] = {0, 0};
  cudaEvent_t pre_ev[2] = {nullptr, nullptr};
  void* pre_dev = nullptr;
  size_t pre_dev_bytes = 0;

  int fail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    error = buf;
    return code;
  }
};

struct Matches {
  Context* ctx = nullptr;
  size_t pts_bytes = 0, segs_bytes = 0;
  float4* pts = nullptr;   // [rounds*32]
  int4* segs = nullptr;    // [nseg+1]
  std::vector<int4> host_segs;  // host copy of segs (the launch checks per-CTA segment counts against it: ggs_lean_fits)
  int nseg = 0;
  int rounds = 0;
  int layout = 0;          // kLayoutPlain / kLayoutPaired (ggs_layout.cuh)
  long long m_total = 0;
  int frames = 0;
  int height = 0, width = 0;
};

#define PDB_CUDA(ctx, call)                                                                          \
  do {                                                                                               \
    cudaError_t err__ = (call);                                                                      \
    if (err__ != cudaSuccess)                                                                        \
      return (ctx)->fail(PDB_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(err__), __FILE__, __LINE__); \
  } while (0)

struct ScopedTimer {  // records an event pair around a launch when profiling is on
  Context* ctx; cudaStream_t st; cudaEvent_t a = nullptr, b = nullptr; int kind;
  ScopedTimer(Context* c, cudaStream_t s, int k) : ctx(c), st(s), kind(k) {
    if (ctx->profiling) { cudaEventCreate(&a); cudaEventCreate(&b); cudaEventRecord(a, st); }
  }
  ~ScopedTimer() {
    if (a) { cudaEventRecord(b, st); ctx->timed.push_back({a, b, kind}); }
  }
};

inline int ensure_buffer(Context* ctx, void** ptr, size_t* have, size_t need) {
  if (*have >= need) return PDB_OK;
  if (*ptr) cudaFree(*ptr);
  *ptr = nullptr;
  *have = 0;
  size_t grow = need + need / 4 + 4096;
  PDB_CUDA(ctx, cudaMalloc(ptr, grow));
  *have = grow;
  return PDB_OK;
}

inline int pool_take(Context* ctx, void** ptr, size_t* got, size_t need) {
  int best = -1;
  for (int i = 0; i < (int)ctx->pool.size(); ++i)
    if (ctx->pool[i].second >= need && (best < 0 || ctx->pool[i].second < ctx->pool[best].second)) best = i;
  if (best >= 0 && ctx->pool[best].second <= 2 * need + 4096) {
    *ptr = ctx->pool[best].first;
    *got = ctx->pool[best].second;
    ctx->pool.erase(ctx->pool.begin() + best);
    return PDB_OK;
  }
  PDB_CUDA(ctx, cudaMalloc(ptr, need));
  *got = need;
  return PDB_OK;
}
inline void pool_give(Context* ctx, void* ptr, size_t bytes) {
  if (!ptr) return;
  if (ctx->pool.size() < 16) ctx->pool.emplace_back(ptr, bytes);
  else cudaFree(ptr);
}

}  // namespace pdb
