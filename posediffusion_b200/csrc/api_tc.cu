// Tensor-core (wgmma + TMA) linear layer: host side (tensor maps, launch) and a test entry point.
#include <cuda.h>
#include <cudaTypedefs.h>

#include <algorithm>
#include <cstdint>
#include <cstdlib>

#include "context.cuh"
#include "tc_linear.cuh"

using namespace pdb;

namespace {

PFN_cuTensorMapEncodeTiled_v12000 get_encode() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  }
  return fn;
}

// Kernel launch, optionally as a programmatic dependent of the previous launch in the stream (csrc/common.cuh: pdl_wait /
// pdl_trigger).  Inside a stream capture this becomes a programmatic edge of the graph.
template <typename... KArgs, typename... Args>
cudaError_t launch_chained(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool pdl, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

// 2-D fp32 row-major [rows, K] tensor, box = box_rows x 32 floats (128 bytes), 128-byte swizzle, zero fill out of bounds
int make_map(Context* ctx, CUtensorMap* map, const float* ptr, int rows, int K, int box_rows) {
  auto encode = get_encode();
  if (!encode) return ctx->fail(PDB_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)K * sizeof(float)};
  cuuint32_t box[2] = {(cuuint32_t)kTcBK, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(ptr), dims, strides, box, estr,
                      CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return ctx->fail(PDB_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d)", (int)r);
  return PDB_OK;
}

}  // namespace

namespace pdb {

// Persistent grid: as many CTAs as are resident on the GPU at once (shared memory and registers decide).  Kernel and
// shared-memory size are fixed per instantiation, so the answer is cached by the caller.
template <typename Kernel>
static int resident_ctas(const Context* ctx, Kernel kernel, size_t smem) {
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kTcThreads, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
  return per_sm * ctx->sm_count;
}

// Y = epilogue(X[S,K] @ W[O,K]^T) on the tensor cores.  K % 32 == 0, O % 64 == 0, all pointers 16-byte aligned.
template <int BN, int ST>
static int launch_tc_linear(Context* ctx, const float* X, const float* W, const TcEpilogue& E, bool& attr, cudaStream_t st) {
  CUtensorMap mx, mw;
  if (int rc = make_map(ctx, &mx, X, E.S, E.K, kTcBM)) return rc;
  if (int rc = make_map(ctx, &mw, W, E.O, E.K, BN)) return rc;
  const size_t smem = tc_smem_bytes(BN, ST);
  static int resident = 0;
  if (!attr) {
    PDB_CUDA(ctx, cudaFuncSetAttribute(tc_linear_kernel<BN, ST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    resident = resident_ctas(ctx, tc_linear_kernel<BN, ST>, smem);
    attr = true;
  }
  const int tiles = (E.O / BN) * ((E.S + kTcBM - 1) / kTcBM) * (E.splits > 1 ? E.splits : 1);
  const int grid = std::min(tiles, resident);
  {
    ScopedTimer timer(ctx, st, 1);
    PDB_CUDA(ctx, launch_chained(tc_linear_kernel<BN, ST>, dim3(grid), dim3(kTcThreads), smem, st, E.pdl != 0, mx, mw, E));
  }
  PDB_CUDA(ctx, cudaGetLastError());
  ctx->launches += 1;
  return PDB_OK;
}

// Swap-AB launch (few tokens): weights on the 128-row M side, NT tokens on the N side (tc_linear.cuh header).
template <int NT>
static int launch_tc_linear_swap(Context* ctx, const float* X, const float* W, const TcEpilogue& E, bool& attr, cudaStream_t st) {
  CUtensorMap mx, mw;
  if (int rc = make_map(ctx, &mx, X, E.S, E.K, NT)) return rc;
  if (int rc = make_map(ctx, &mw, W, E.O, E.K, kTcBM)) return rc;
  const size_t smem = tc_smem_bytes(NT, kTcStages);
  static int resident = 0;
  if (!attr) {
    PDB_CUDA(ctx, (cudaFuncSetAttribute(tc_linear_kernel<NT, kTcStages, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)));
    resident = resident_ctas(ctx, tc_linear_kernel<NT, kTcStages, true>, smem);
    attr = true;
  }
  const int tiles = (E.O / kTcBM) * ((E.S + NT - 1) / NT);
  const int grid = std::min(tiles, resident);
  {
    ScopedTimer timer(ctx, st, 1);
    tc_linear_kernel<NT, kTcStages, true><<<grid, kTcThreads, smem, st>>>(mx, mw, E);
  }
  PDB_CUDA(ctx, cudaGetLastError());
  ctx->launches += 1;
  return PDB_OK;
}

// Swap-AB tiles are taken for at most 96 tokens when enabled (pdb_debug_tc_swap / PDB_TC_SWAP=1).  Default off: without split-K
// only O/128 CTAs stream the weights and the tile is bound by one SM's L2 bandwidth.
static bool tc_linear_swapped(const Context* ctx, int S, int O) {
  static const bool env_on = [] { const char* v = getenv("PDB_TC_SWAP"); return v && v[0] == '1'; }();
  return S <= 96 && O % kTcBM == 0 && (env_on || ctx->tc_swap);
}

// Y = epilogue(X[S,K] @ W[O,K]^T) on the tensor cores.  K % 32 == 0, O % 64 == 0, all pointers 16-byte aligned.
// 128-feature tiles (two wgmma 64x128x8 per K-step) when they still fill the machine, 64-feature tiles for the small-S denoiser shapes,
// swap-AB tiles (weights on the M side) for at most 96 tokens when enabled (pdb_debug_tc_swap / PDB_TC_SWAP=1).
int enqueue_tc_linear(Context* ctx, const float* X, const float* W, TcEpilogue E, cudaStream_t st) {
  if (E.K % kTcBK || E.O % 64 || E.S < 1) return ctx->fail(PDB_ERR_INVALID, "tc_linear shape (S=%d, O=%d, K=%d)", E.S, E.O, E.K);
  if (tc_linear_swapped(ctx, E.S, E.O)) {
    E.splits = 1;
    E.stats = 0;
    if (E.S <= 32) return launch_tc_linear_swap<32>(ctx, X, W, E, ctx->attr->tc_swap[0], st);
    if (E.S <= 64) return launch_tc_linear_swap<64>(ctx, X, W, E, ctx->attr->tc_swap[1], st);
    return launch_tc_linear_swap<96>(ctx, X, W, E, ctx->attr->tc_swap[2], st);
  }
  const long long wide_tiles = (long long)(E.O / 128) * ((E.S + kTcBM - 1) / kTcBM);
  if (E.O % 128 == 0 && wide_tiles >= ctx->sm_count) {
    // one CTA per SM (64 accumulator registers per consumer thread): a 6 x 32 KB ring lets the producer run half a K = 384
    // tile ahead while the consumers are in the epilogue
    E.splits = 1;
    E.stats = 0;
    return launch_tc_linear<128, 6>(ctx, X, W, E, ctx->attr->tc128, st);
  }
  if (E.allow_small && tc_linear_small(ctx, E.S, E.O)) {
    // Fewer 64-feature tiles than SMs (the denoiser at a few hundred tokens): a CTA's k-loop is a serial chain of TMA round
    // trips, so (i) an 8-deep ring keeps 192 KB in flight per SM instead of 96, (ii) GEMMs that update the residual stream in
    // place are split along K over the idle SMs, the partial products added to Y with vector reductions, and (iii) the folded
    // LayerNorm statistics come out of the X tiles inside the kernel (E.stats, requested by the caller).
    const int tiles = (E.O / 64) * ((E.S + kTcBM - 1) / kTcBM), num_kb = E.K / kTcBK;
    E.splits = 1;
    const bool in_place = E.residual == E.Y && E.ldr == E.ldy && !E.relu && !E.gelu && !E.colsum;
    if (in_place)
      for (int s : {8, 4, 2})
        if (num_kb % s == 0 && num_kb / s >= 2 && tiles * s <= ctx->sm_count) {
          E.splits = s;
          break;
        }
    if (!E.colsum || E.splits != 1) E.stats = 0;
    return launch_tc_linear<64, 8>(ctx, X, W, E, ctx->attr->tc_deep, st);
  }
  E.splits = 1;
  E.stats = 0;
  return launch_tc_linear<64, kTcStages>(ctx, X, W, E, ctx->attr->tc, st);
}

// the launcher's "small problem" regime (see above); callers that want in-kernel LayerNorm statistics ask first
bool tc_linear_small(const Context* ctx, int S, int O) {
  if (tc_linear_swapped(ctx, S, O)) return false;
  return (long long)(O / 64) * ((S + kTcBM - 1) / kTcBM) <= ctx->sm_count && !getenv("PDB_TC_NO_SMALL");
}

}  // namespace pdb

extern "C" int pdb_debug_tc_linear(pdb_context* c, const float* x_dev, const float* w_dev, const float* bias_dev,
                                   const float* residual_dev, float* y_dev, int32_t S, int32_t O, int32_t K, int32_t relu,
                                   void* stream) {
  if (!c) return PDB_ERR_INVALID;
  Context* ctx = reinterpret_cast<Context*>(c);
  if (!x_dev || !w_dev || !y_dev) return ctx->fail(PDB_ERR_INVALID, "null argument");
  PDB_CUDA(ctx, cudaSetDevice(ctx->device));
  TcEpilogue E = {};
  E.bias = bias_dev;
  E.residual = residual_dev;
  E.ldr = O;
  E.Y = y_dev;
  E.ldy = O;
  E.S = S;
  E.O = O;
  E.K = K;
  E.relu = relu;
  E.allow_small = 1;
  return enqueue_tc_linear(ctx, x_dev, w_dev, E, static_cast<cudaStream_t>(stream));
}

// ================================================================================================
// Tensor-core denoiser engine (S >= 128 tokens per GPU): one kernel per stage, projections on wgmma/TMA tiles.
// Same maths as denoiser_kernel (csrc/denoiser.cuh); LayerNorm is folded into the QKV / FF1 weights at load time and
// applied in the GEMM epilogue from per-row statistics.  TF32 products, fp32 accumulate / residual stream.
// ================================================================================================
#include "weights.cuh"

namespace {

__global__ void embed_kernel(const float* __restrict__ x, float* __restrict__ emb, int S) {  // [S,9] -> [S,256] harmonic features
  pdl_trigger();
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= S * kPoseEmbPad) return;
  const int s = i / kPoseEmbPad, col = i - s * kPoseEmbPad;
  float v = 0.f;
  if (col < 180) {
    const int j = col < 90 ? col : col - 90;
    const int c = j / 10, k = j - c * 10;
    const float arg = x[s * 9 + c] * (float)(1 << k);
    v = col < 90 ? sinf(arg) : cosf(arg);
  } else if (col < kPoseEmb) {
    v = x[s * 9 + (col - 180)];
  }
  emb[i] = v;
}
__global__ void pivot_add_kernel(float* __restrict__ zproj, const float* __restrict__ w_pivot, int batch, int frames) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // first frame of every sequence gets the pivot column
  if (i < batch * kDM) zproj[(size_t)(i / kDM) * frames * kDM + (i % kDM)] += w_pivot[i % kDM];
}
__global__ void row_stats_kernel(const float* __restrict__ h, float* __restrict__ mean, float* __restrict__ rstd, int S) {
  pdl_trigger();
  pdl_wait();
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= S) return;
  const float4* p = reinterpret_cast<const float4*>(h + (size_t)row * kDM);
  float4 v[4];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    v[i] = p[lane + 32 * i];
    sum += v[i].x + v[i].y + v[i].z + v[i].w;
  }
  const float m = warp_sum(sum) * (1.0f / kDM);
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float a = v[i].x - m, b = v[i].y - m, c = v[i].z - m, d = v[i].w - m;
    sq += a * a + b * b + c * c + d * d;
  }
  const float var = warp_sum(sq) * (1.0f / kDM);
  if (lane == 0) {
    mean[row] = m;
    rstd[row] = 1.0f / sqrtf(var + kLnEps);
  }
}
__global__ void __launch_bounds__(kDenThreads) attention_kernel(const float* __restrict__ qkv, float* __restrict__ att, int frames) {
  extern __shared__ __align__(16) float att_smem[];
  pdl_trigger();
  pdl_wait();
  const int chunks = (frames + kDenWarps - 1) / kDenWarps;
  const int item = blockIdx.x;
  attention_item<false>(att_smem, qkv, att, item / (kHeads * chunks), (item / chunks) % kHeads, item % chunks, frames, 0u, 0u);
}
// the timestep lives on the device (tstate = {t, t_lo}) so that one captured graph serves every diffusion step
__global__ void __launch_bounds__(kDenThreads) tail_kernel(const __grid_constant__ DenoiserDev W, const __grid_constant__ DenoiserRun R, const int* __restrict__ tstate) {
  pdl_trigger();
  pdl_wait();
  const int s = blockIdx.x * kDenWarps + (threadIdx.x >> 5);
  const int t = tstate[0];
  if (s < R.tokens) tail_token<false>(W, R, s, t, t == tstate[1], 0u, 0u);
}
__global__ void step_set_kernel(int* tstate, int t, int t_lo) { tstate[0] = t; tstate[1] = t_lo; }
__global__ void step_dec_kernel(int* tstate) {
  pdl_wait();
  tstate[0] -= 1;
}

}  // namespace

namespace pdb {

// `dev` is the loaded weights' descriptor, or its copy with a DDIM prefix's per-timestep tables (tproj, sched; api_sampler.cu).
int enqueue_denoiser_tc(Context* ctx, const DenoiserDev& dev, DenoiserRun run, cudaStream_t st) {
  const DenoiserWeights* w = ctx->weights;
  const TcWeights& T = w->tc;
  const int S = run.tokens, B = run.batch, N = run.frames;
  const size_t need = sizeof(float) * (denoiser_ws_floats(S) + (size_t)S * (kPoseEmbPad + 2) + 64);
  if (int rc = ensure_buffer(ctx, &ctx->den_ws, &ctx->den_ws_bytes, need)) return rc;
  int* tstate = reinterpret_cast<int*>(ctx->den_ws) + 32;  // words 32..33 of the 256-byte header (0 = barrier counter)
  float* ws = static_cast<float*>(ctx->den_ws) + 64;
  run.zproj = ws; ws += (size_t)S * kDM;
  run.h = ws;     ws += (size_t)S * kDM;
  run.qkv = ws;   ws += (size_t)S * 3 * kDM;
  run.att = ws;   ws += (size_t)S * kDM;
  run.ff = ws;    ws += (size_t)S * kFF;
  run.u = ws;     ws += (size_t)S * kHid;
  float* emb = ws; ws += (size_t)S * kPoseEmbPad;
  float* mean = ws; ws += S;
  float* rstd = ws;
  bool pdl = false;  // set while a step is being enqueued
  auto lin = [&](const float* X, const float* Wm, int O, int K, const float* bias, const int* t_ptr, const float* residual, int ldr,
                 const float* colsum, float* Y, int relu, cudaStream_t s) {
    TcEpilogue E = {};
    E.bias = bias; E.t_ptr = t_ptr; E.bias_t_stride = kDM; E.residual = residual; E.ldr = ldr;
    E.colsum = colsum; E.row_mean = colsum ? mean : nullptr; E.row_rstd = colsum ? rstd : nullptr;
    E.Y = Y; E.ldy = O; E.S = S; E.O = O; E.K = K; E.relu = relu;
    E.allow_small = 1;
    E.pdl = pdl;
    E.stats = colsum && tc_linear_small(ctx, S, O);  // then no row_stats_kernel precedes this GEMM (below)
    return enqueue_tc_linear(ctx, X, Wm, E, s);
  };
  const size_t att_smem = sizeof(float) * ((size_t)N * (kHD + 4) + (size_t)N * kHD + 2 * kDenWarps * kHD) + 64;
  size_t& att_attr = ctx->attr->att;
  if (att_smem > att_attr) {
    PDB_CUDA(ctx, cudaFuncSetAttribute(attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)att_smem));
    att_attr = att_smem;
  }
  const int chunks = (N + kDenWarps - 1) / kDenWarps;
  const bool was_profiling = ctx->profiling;
  ScopedTimer total(ctx, st, 1);  // one event pair around the whole call (events cannot be recorded inside the capture)
  ctx->profiling = false;
  if (run.compute_zproj) {
    if (int rc = lin(run.z, T.wz, kDM, kZ, T.b_first, nullptr, nullptr, 0, nullptr, run.zproj, 0, st)) { ctx->profiling = was_profiling; return rc; }
    pivot_add_kernel<<<(B * kDM + 255) / 256, 256, 0, st>>>(run.zproj, T.w_pivot, B, N);
    ctx->launches += 1;
  }
  // ---- one diffusion step = 60 launches (44 when the LayerNorm statistics are computed inside the QKV / FF1 GEMMs);
  // captured once per buffer set, replayed per step ----
  const bool stats_qkv = tc_linear_small(ctx, S, 3 * kDM), stats_ff1 = tc_linear_small(ctx, S, kFF);
  auto enqueue_step = [&](cudaStream_t s) -> int {
    // the kernels of a step form one programmatic chain (the first one has no predecessor in the capture); only small steps
    // gain from overlapping a kernel's prologue with its predecessor's tail
    pdl = ctx->tc_pdl && S <= 320;
    PDB_CUDA(ctx, launch_chained(embed_kernel, dim3((S * kPoseEmbPad + 255) / 256), dim3(256), 0, s, false, (const float*)run.x, emb, S));
    if (int rc = lin(emb, T.wx, kDM, kPoseEmbPad, dev.tproj, tstate, run.zproj, kDM, nullptr, run.h, 0, s)) return rc;
    for (int l = 0; l < kLayers; ++l) {
      const TcLayer& L = T.layer[l];
      if (!stats_qkv) PDB_CUDA(ctx, launch_chained(row_stats_kernel, dim3((S + 7) / 8), dim3(256), 0, s, pdl, (const float*)run.h, mean, rstd, S));
      if (int rc = lin(run.h, L.wqkv, 3 * kDM, kDM, L.bias_qkv, nullptr, nullptr, 0, L.colsum_qkv, run.qkv, 0, s)) return rc;
      PDB_CUDA(ctx, launch_chained(attention_kernel, dim3(B * kHeads * chunks), dim3(kDenThreads), att_smem, s, pdl, (const float*)run.qkv, run.att, N));
      if (int rc = lin(run.att, L.wout, kDM, kDM, L.bout, nullptr, run.h, kDM, nullptr, run.h, 0, s)) return rc;
      if (!stats_ff1) PDB_CUDA(ctx, launch_chained(row_stats_kernel, dim3((S + 7) / 8), dim3(256), 0, s, pdl, (const float*)run.h, mean, rstd, S));
      if (int rc = lin(run.h, L.wff1, kFF, kDM, L.bias_ff1, nullptr, nullptr, 0, L.colsum_ff1, run.ff, 1, s)) return rc;
      if (int rc = lin(run.ff, L.wff2, kDM, kFF, L.bff2, nullptr, run.h, kDM, nullptr, run.h, 0, s)) return rc;
    }
    if (int rc = lin(run.h, T.wlast0, kHid, kDM, T.blast0, nullptr, nullptr, 0, nullptr, run.u, 0, s)) return rc;
    PDB_CUDA(ctx, launch_chained(tail_kernel, dim3((S + kDenWarps - 1) / kDenWarps), dim3(kDenThreads), 0, s, pdl, dev, run, (const int*)tstate));
    PDB_CUDA(ctx, launch_chained(step_dec_kernel, dim3(1), dim3(1), 0, s, pdl, tstate));
    pdl = false;
    return PDB_OK;
  };
  const int kNodes = 2 + kLayers * (7 - (stats_qkv ? 1 : 0) - (stats_ff1 ? 1 : 0)) + 3;
  std::vector<size_t> key = {(size_t)S, (size_t)B, (size_t)N, (size_t)run.guide_below, (size_t)ctx->den_ws, (size_t)run.x,
                             (size_t)run.draws, (size_t)run.trail, (size_t)run.eps_out, (size_t)run.x0_out, (size_t)run.mean_out,
                             (size_t)w->tc_arena, (size_t)dev.tproj, (size_t)dev.sched, (size_t)ctx->tc_swap, (size_t)stats_qkv, (size_t)stats_ff1,
                             (size_t)tc_linear_small(ctx, S, kDM), (size_t)(ctx->tc_pdl && S <= 320)};  // launcher regime: the captured kernels differ
  if (!ctx->tc_graph || ctx->tc_graph_key != key) {
    if (ctx->tc_graph) { cudaGraphExecDestroy(ctx->tc_graph); ctx->tc_graph = nullptr; }
    if (!ctx->tc_capture_stream) PDB_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->tc_capture_stream, cudaStreamNonBlocking));
    const long long before = ctx->launches;
    cudaGraph_t graph = nullptr;
    PDB_CUDA(ctx, cudaStreamBeginCapture(ctx->tc_capture_stream, cudaStreamCaptureModeThreadLocal));
    const int rc = enqueue_step(ctx->tc_capture_stream);
    cudaError_t err = cudaStreamEndCapture(ctx->tc_capture_stream, &graph);
    ctx->launches = before;  // nothing ran yet
    if (rc != PDB_OK || err != cudaSuccess) {
      if (graph) cudaGraphDestroy(graph);
      ctx->profiling = was_profiling;
      return rc != PDB_OK ? rc : ctx->fail(PDB_ERR_CUDA, "graph capture failed: %s", cudaGetErrorString(err));
    }
    err = cudaGraphInstantiate(&ctx->tc_graph, graph, 0);
    cudaGraphDestroy(graph);
    if (err != cudaSuccess) {
      ctx->tc_graph = nullptr;
      ctx->profiling = was_profiling;
      return ctx->fail(PDB_ERR_CUDA, "graph instantiate failed: %s", cudaGetErrorString(err));
    }
    ctx->tc_graph_key = key;
    ctx->tc_graph_nodes = kNodes;
  }
  step_set_kernel<<<1, 1, 0, st>>>(tstate, run.t_hi, run.t_lo);
  for (int t = run.t_hi; t >= run.t_lo; --t) {
    cudaError_t err = cudaGraphLaunch(ctx->tc_graph, st);
    if (err != cudaSuccess) {
      ctx->profiling = was_profiling;
      return ctx->fail(PDB_ERR_CUDA, "graph launch failed: %s", cudaGetErrorString(err));
    }
  }
  ctx->launches += 1 + (long long)kNodes * (run.t_hi - run.t_lo + 1);
  ctx->profiling = was_profiling;
  PDB_CUDA(ctx, cudaGetLastError());
  return PDB_OK;
}

}  // namespace pdb

extern "C" int pdb_debug_tc_swap(pdb_context* c, int32_t on) {
  if (!c) return PDB_ERR_INVALID;
  reinterpret_cast<Context*>(c)->tc_swap = on != 0;
  return PDB_OK;
}

extern "C" int pdb_denoiser_engine(pdb_context* c, int32_t mode) {
  if (!c || mode < 0 || mode > 2) return PDB_ERR_INVALID;
  reinterpret_cast<Context*>(c)->denoiser_engine = mode;
  return PDB_OK;
}

extern "C" int pdb_debug_denoiser_handover(pdb_context* c, int32_t flagged) {
  if (!c) return PDB_ERR_INVALID;
  reinterpret_cast<Context*>(c)->den_flag = flagged != 0;
  return PDB_OK;
}
