// C-ABI entry points: denoiser weights, denoiser forward, p_sample, p_sample_loop (device and host buffers).
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <new>
#include <vector>

#include "context.cuh"
#include "denoiser.cuh"
#include "fold_ln.cuh"
#include "weights.cuh"

using namespace pdb;

namespace pdb {
int enqueue_ggs(Context* ctx, pdb_matches* const* problems, int batch, int frames, float* pose_dev, const pdb_ggs_config* cfg,
                pdb_ggs_stats* stats_dev, cudaStream_t st);
int check_ggs_problems(Context* ctx, pdb_matches* const* problems, int batch, int frames);

int enqueue_denoiser_tc(Context* ctx, DenoiserRun run, cudaStream_t st);
void vit_release(Context* ctx);
}  // namespace pdb

constexpr int kTcMinTokens = 128;

namespace {

// ---- one-off kernels used at weight-load time (not on the hot path) ----
// W [O][ldw] row-major (column window [c0, c0+Kuse)) -> Wp [Kpad/4][O] float4, zero padded
__global__ void pack_k4_kernel(const float* __restrict__ W, int O, int ldw, int c0, int Kuse, int Kpad, float4* __restrict__ Wp) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (Kpad / 4) * O) return;
  const int k4 = idx / O, o = idx - k4 * O;
  float v[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int k = k4 * 4 + j;
    v[j] = (k < Kuse) ? W[(size_t)o * ldw + c0 + k] : 0.f;
  }
  Wp[idx] = make_float4(v[0], v[1], v[2], v[3]);
}
__global__ void gather_col_kernel(const float* __restrict__ W, int O, int ldw, int col, float* __restrict__ out) {
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o < O) out[o] = W[(size_t)o * ldw + col];
}
// Y[s][o] = act(sum_k X[s][k] * W[o][c0+k] + bias[o]); sequential fp32 sum (load-time table only)
__global__ void naive_linear_kernel(const float* __restrict__ X, int S, int K, const float* __restrict__ W, int O, int ldw,
                                    int c0, const float* __restrict__ bias, float* __restrict__ Y, int silu) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= S * O) return;
  const int s = idx / O, o = idx - s * O;
  float acc = 0.f;
  for (int k = 0; k < K; ++k) acc = fmaf(X[(size_t)s * K + k], W[(size_t)o * ldw + c0 + k], acc);
  if (bias) acc += bias[o];
  if (silu) acc = acc / (1.0f + expf(-acc));
  Y[idx] = acc;
}

// W[O][ldw] column window -> dense row-major [O][Kpad] (zero padded): operands of the tensor-core engine
__global__ void copy_cols_kernel(const float* __restrict__ W, int O, int ldw, int c0, int Kuse, int Kpad, float* __restrict__ out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= O * Kpad) return;
  const int o = idx / Kpad, k = idx - o * Kpad;
  out[idx] = (k < Kuse) ? W[(size_t)o * ldw + c0 + k] : 0.f;
}
const int kShape[6][2] = {{128, 256}, {128, 0}, {128, 128}, {128, 0}, {512, 702}, {512, 0}};

size_t tensor_floats(int i) {
  if (i < 6) return (size_t)kShape[i][0] * (kShape[i][1] ? kShape[i][1] : 1);
  if (i < 6 + 12 * kLayers) {
    switch ((i - 6) % 12) {
      case 0: return 1536 * 512;
      case 1: return 1536;
      case 2: return 512 * 512;
      case 3: return 512;
      case 4: return 1024 * 512;
      case 5: return 1024;
      case 6: return 512 * 1024;
      case 7: return 512;
      default: return 512;
    }
  }
  switch (i - (6 + 12 * kLayers)) {
    case 0: return 128 * 512;
    case 1: return 128;
    case 2: return 128;
    case 3: return 128;
    case 4: return 9 * 128;
    default: return 9;
  }
}

int pick_token_tile(int tokens) {
  const int cand[5] = {8, 16, 20, 24, 32};  // 20 = the headline sequence length (no padded token rows)
  int best = 32, best_pad = 1 << 30;
  for (int c : cand) {
    const int pad = (tokens + c - 1) / c * c;
    if (pad < best_pad || (pad == best_pad && c > best)) {
      best = c;
      best_pad = pad;
    }
  }
  return best;
}

template <int TS, bool kFlag>
int launch_denoiser(Context* ctx, const DenoiserRun& run, int grid, cudaStream_t st) {
  const size_t smem = denoiser_smem_bytes(TS, run.frames);
  if (smem > ctx->smem_optin) return ctx->fail(PDB_ERR_LIMIT, "denoiser needs %zu B shared memory", smem);
  size_t& attr_bytes = ctx->attr_den[(kFlag ? 8 : 0) + TS / 4 - 1];  // static shared memory counts against the opt-in limit: ask for what we use
  if (smem > attr_bytes) {
    PDB_CUDA(ctx, cudaFuncSetAttribute(denoiser_kernel<TS, kFlag>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_bytes = smem;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(kDenThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  {
    ScopedTimer timer(ctx, st, 1);
    PDB_CUDA(ctx, cudaLaunchKernelEx(&cfg, denoiser_kernel<TS, kFlag>, ctx->weights->dev, run));
  }
  ctx->launches += 1;
  return PDB_OK;
}

// Fill the workspace pointers of `run` and launch steps t_hi..t_lo.
int enqueue_denoiser(Context* ctx, DenoiserRun run, cudaStream_t st) {
  if (!ctx->weights) return ctx->fail(PDB_ERR_STATE, "denoiser weights not loaded (pdb_denoiser_load)");
  if (run.batch < 1 || run.frames < 1) return ctx->fail(PDB_ERR_INVALID, "empty batch");
  if (run.frames > PDB_MAX_FRAMES) return ctx->fail(PDB_ERR_LIMIT, "frames %d > PDB_MAX_FRAMES", run.frames);
  if (run.t_hi >= kT || run.t_lo < 0 || run.t_hi < run.t_lo) return ctx->fail(PDB_ERR_INVALID, "bad timestep range");
  const int S = run.batch * run.frames;
  run.tokens = S;
  // engine: exact-fp32 persistent kernel below kTcMinTokens tokens (latency bound), wgmma/TMA tiles (TF32 products) at or
  // above it (throughput bound).  ctx->denoiser_engine: 0 auto, 1 force fp32, 2 force tensor cores.
  const bool use_tc = ctx->denoiser_engine == 2 || (ctx->denoiser_engine == 0 && S >= kTcMinTokens);
  if (use_tc) return enqueue_denoiser_tc(ctx, run, st);
  const size_t need = sizeof(float) * denoiser_ws_floats(S);
  if (int rc = ensure_buffer(ctx, &ctx->den_ws, &ctx->den_ws_bytes, need)) return rc;
  float* ws = static_cast<float*>(ctx->den_ws);
  run.bar = reinterpret_cast<unsigned*>(ws);
  ws += 64;
  run.zproj = ws; ws += (size_t)S * kDM;
  run.h = ws;     ws += (size_t)S * kDM;
  run.qkv = ws;   ws += (size_t)S * 3 * kDM;
  run.att = ws;   ws += (size_t)S * kDM;
  run.ff = ws;    ws += (size_t)S * kFF;
  run.u = ws;
  PDB_CUDA(ctx, cudaMemsetAsync(run.bar, 0, 256, st));
  // stage hand-over: group barriers, or flag-carrying activation words (no barriers) when pdb_debug_denoiser_handover /
  // PDB_DEN_FLAG=1 selects that instantiation (measured slower, kept as a tested alternative)
  const bool flagged = ctx->den_flag != 0;
  if (flagged) {
    const size_t words = denoiser_flag_ws_words(S);
    const unsigned tags = (unsigned)(run.t_hi - run.t_lo + 1) * kTagsPerStep;
    const bool fresh = ctx->den_flag_ws_bytes < sizeof(unsigned long long) * words;
    if (int rc = ensure_buffer(ctx, &ctx->den_flag_ws, &ctx->den_flag_ws_bytes, sizeof(unsigned long long) * words)) return rc;
    if (fresh || ctx->den_tag > 0xffffffffu - tags - 1u) {  // new buffer, or the 32-bit versions would wrap: start over from tag 1
      PDB_CUDA(ctx, cudaMemsetAsync(ctx->den_flag_ws, 0, ctx->den_flag_ws_bytes, st));
      ctx->den_tag = 1u;
    }
    unsigned long long* fw = static_cast<unsigned long long*>(ctx->den_flag_ws);
    run.fh = fw;   fw += (size_t)S * kDM;
    run.fqkv = fw; fw += (size_t)S * 2 * 3 * kDM;
    run.fatt = fw; fw += (size_t)S * kDM;
    run.fff = fw;  fw += (size_t)S * kFF;
    run.fu = fw;   fw += (size_t)S * kHid;
    run.fx = fw;
    run.tag_base = ctx->den_tag;
    ctx->den_tag += tags;
  }
  run.dbg_clock = ctx->den_clock ? ctx->ggs_clock : nullptr;  // pdb_debug_ggs_clocks(enable = 2): probe the denoiser instead
  const int TS = pick_token_tile(S);
  const int tiles = (S + TS - 1) / TS;
  int grid = tiles * (3 * kDM / kFPI);  // widest stage (QKV)
  if (grid > ctx->sm_count) grid = ctx->sm_count;
  if (const char* g = getenv("PDB_DEN_GRID")) {  // tuning knob: number of CTAs of the persistent denoiser kernel
    const int v = atoi(g);
    if (v >= 1 && v < grid) grid = v;
  }
  if (flagged) {
    switch (TS) {
      case 8: return launch_denoiser<8, true>(ctx, run, grid, st);
      case 16: return launch_denoiser<16, true>(ctx, run, grid, st);
      case 20: return launch_denoiser<20, true>(ctx, run, grid, st);
      case 24: return launch_denoiser<24, true>(ctx, run, grid, st);
      default: return launch_denoiser<32, true>(ctx, run, grid, st);
    }
  }
  switch (TS) {
    case 8: return launch_denoiser<8, false>(ctx, run, grid, st);
    case 16: return launch_denoiser<16, false>(ctx, run, grid, st);
    case 20: return launch_denoiser<20, false>(ctx, run, grid, st);
    case 24: return launch_denoiser<24, false>(ctx, run, grid, st);
    default: return launch_denoiser<32, false>(ctx, run, grid, st);
  }
}

// The sampling loop in two halves, so that a caller can do host work (match packing) between them while the first half runs:
// loop_prefix enqueues x_T = draws[0] (gaussian_diffuser.py:289) and the unguided steps t = T-1 .. guide_below in ONE launch,
// loop_guided the guided steps (denoiser -> posterior mean -> GGS in place).
struct LoopState {
  DenoiserRun run = {};
  int guide_below = 0;
  bool first = true;
  size_t n = 0;
  float* pose = nullptr;
  float* trail = nullptr;
};

int loop_prefix(Context* ctx, const float* z_dev, const float* draws_dev, int batch, int frames, int guide_below, float* pose_dev,
                float* trail_dev, cudaStream_t st, LoopState* loop) {
  if (guide_below > kT) guide_below = kT;
  if (guide_below < 0) guide_below = 0;
  const size_t n = (size_t)batch * frames * kTargetDim;
  PDB_CUDA(ctx, cudaMemcpyAsync(pose_dev, draws_dev, sizeof(float) * n, cudaMemcpyDeviceToDevice, st));
  if (trail_dev) PDB_CUDA(ctx, cudaMemcpyAsync(trail_dev, draws_dev, sizeof(float) * n, cudaMemcpyDeviceToDevice, st));
  loop->n = n;
  loop->guide_below = guide_below;
  loop->pose = pose_dev;
  loop->trail = trail_dev;
  DenoiserRun& run = loop->run;
  run.batch = batch; run.frames = frames;
  run.guide_below = guide_below;
  run.x = pose_dev; run.z = z_dev; run.draws = draws_dev; run.trail = trail_dev;
  if (guide_below < kT) {
    run.t_hi = kT - 1; run.t_lo = guide_below;
    run.compute_zproj = 1;
    if (int rc = enqueue_denoiser(ctx, run, st)) return rc;
    loop->first = false;
  }
  return PDB_OK;
}

int loop_guided(Context* ctx, LoopState* loop, pdb_matches* const* problems, const pdb_ggs_config* cfg, pdb_ggs_stats* stats_dev,
                cudaStream_t st) {
  DenoiserRun& run = loop->run;
  for (int t = loop->guide_below - 1; t >= 0; --t) {
    run.t_hi = run.t_lo = t;
    run.compute_zproj = loop->first ? 1 : 0;
    loop->first = false;
    if (int rc = enqueue_denoiser(ctx, run, st)) return rc;
    pdb_ggs_stats* stats = stats_dev ? stats_dev + (size_t)(loop->guide_below - 1 - t) * run.batch : nullptr;
    if (int rc = enqueue_ggs(ctx, problems, run.batch, run.frames, loop->pose, cfg, stats, st)) return rc;
    if (loop->trail)
      PDB_CUDA(ctx, cudaMemcpyAsync(loop->trail + (size_t)(kT - t) * loop->n, loop->pose, sizeof(float) * loop->n,
                                    cudaMemcpyDeviceToDevice, st));
  }
  return PDB_OK;
}

}  // namespace

extern "C" {

void pdb_destroy(pdb_context* c) {
  if (!c) return;
  Context* ctx = reinterpret_cast<Context*>(c);
  cudaSetDevice(ctx->device);
  if (ctx->weights) {
    if (ctx->weights->arena) cudaFree(ctx->weights->arena);
    if (ctx->weights->raw) cudaFree(ctx->weights->raw);
    if (ctx->weights->tc_arena) cudaFree(ctx->weights->tc_arena);
    delete ctx->weights;
  }
  vit_release(ctx);
  if (ctx->ggs_ws) cudaFree(ctx->ggs_ws);
  if (ctx->den_ws) cudaFree(ctx->den_ws);
  if (ctx->den_flag_ws) cudaFree(ctx->den_flag_ws);
  if (ctx->stage) cudaFree(ctx->stage);
  if (ctx->tc_graph) cudaGraphExecDestroy(ctx->tc_graph);
  if (ctx->tc_capture_stream) cudaStreamDestroy(ctx->tc_capture_stream);
  if (ctx->pack_stream) cudaStreamDestroy(ctx->pack_stream);
  for (auto& b : ctx->pool) cudaFree(b.first);
  if (ctx->pin) cudaFreeHost(ctx->pin);
  for (int s = 0; s < 2; ++s) {
    if (ctx->pre_pin[s]) cudaFreeHost(ctx->pre_pin[s]);
    if (ctx->pre_ev[s]) cudaEventDestroy(ctx->pre_ev[s]);
  }
  if (ctx->pre_dev) cudaFree(ctx->pre_dev);
  if (ctx->ggs_clock) cudaFree(ctx->ggs_clock);
  delete ctx;
}

// DDPM schedule exactly as GaussianDiffusion.init_diff_hyper builds it (gaussian_diffuser.py:136-187):
// float64 linspace / cumprod, cast to float32.  Host only (no GPU needed): out[100][8] =
// {sqrt_recip_alphas_cumprod, sqrt_recipm1_alphas_cumprod, posterior_mean_coef1, posterior_mean_coef2,
//  exp(0.5 * posterior_log_variance_clipped), posterior_log_variance_clipped, betas, alphas_cumprod}
int pdb_schedule_table(float* out, double beta_1, double beta_T) {
  if (!out) return PDB_ERR_INVALID;
  const int n = kT;
  double beta[kT], abar[kT];
  const double step = (beta_T - beta_1) / (double)(n - 1);
  for (int i = 0; i < n; ++i)  // torch.linspace fills symmetrically from both ends
    beta[i] = (i < n / 2) ? beta_1 + step * i : beta_T - step * (n - 1 - i);
  double prod = 1.0;
  for (int i = 0; i < n; ++i) {
    prod *= (1.0 - beta[i]);
    abar[i] = prod;
  }
  for (int i = 0; i < n; ++i) {
    const double prev = i ? abar[i - 1] : 1.0;
    const double pv = beta[i] * (1.0 - prev) / (1.0 - abar[i]);
    const float logv = (float)std::log(pv < 1e-20 ? 1e-20 : pv);
    float* r = out + i * 8;
    r[0] = (float)std::sqrt(1.0 / abar[i]);
    r[1] = (float)std::sqrt(1.0 / abar[i] - 1.0);
    r[2] = (float)(beta[i] * std::sqrt(prev) / (1.0 - abar[i]));
    r[3] = (float)((1.0 - prev) * std::sqrt(1.0 - beta[i]) / (1.0 - abar[i]));
    r[4] = expf(0.5f * logv);
    r[5] = logv;
    r[6] = (float)beta[i];
    r[7] = (float)abar[i];
  }
  return PDB_OK;
}

int pdb_denoiser_load(pdb_context* c, const float* const* tensors, int32_t count, void* stream) {
  if (!c) return PDB_ERR_INVALID;
  Context* ctx = reinterpret_cast<Context*>(c);
  if (!tensors || count != PDB_NUM_WEIGHT_TENSORS)
    return ctx->fail(PDB_ERR_INVALID, "expected %d weight tensors, got %d", PDB_NUM_WEIGHT_TENSORS, count);
  for (int i = 0; i < count; ++i)
    if (!tensors[i]) return ctx->fail(PDB_ERR_INVALID, "weight tensor %d is null", i);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  PDB_CUDA(ctx, cudaSetDevice(ctx->device));
  // raw staging copy of all tensors (host or device source)
  size_t raw_total = 0;
  std::vector<size_t> off(count);
  for (int i = 0; i < count; ++i) {
    off[i] = raw_total;
    raw_total += (tensor_floats(i) + 3) / 4 * 4;
  }
  float* raw = nullptr;
  PDB_CUDA(ctx, cudaMalloc(&raw, sizeof(float) * raw_total));
  for (int i = 0; i < count; ++i) {
    cudaError_t err = cudaMemcpyAsync(raw + off[i], tensors[i], sizeof(float) * tensor_floats(i), cudaMemcpyDefault, st);
    if (err != cudaSuccess) {
      cudaFree(raw);
      return ctx->fail(PDB_ERR_CUDA, "copy of weight tensor %d failed: %s", i, cudaGetErrorString(err));
    }
  }
  // packed arena
  size_t total = 0;
  auto take = [&](size_t n) {
    size_t at = total;
    total += (n + 3) / 4 * 4;
    return at;
  };
  const size_t o_fx = take((size_t)kPoseEmbPad * kDM), o_fz = take((size_t)kZ * kDM), o_piv = take(kDM), o_bf = take(kDM);
  const size_t o_tproj = take((size_t)kT * kDM), o_sched = take((size_t)kT * 8);
  size_t o_l[kLayers][12];
  for (int l = 0; l < kLayers; ++l) {
    o_l[l][0] = take((size_t)kDM * 3 * kDM); o_l[l][1] = take(3 * kDM);
    o_l[l][2] = take((size_t)kDM * kDM);     o_l[l][3] = take(kDM);
    o_l[l][4] = take((size_t)kDM * kFF);     o_l[l][5] = take(kFF);
    o_l[l][6] = take((size_t)kFF * kDM);     o_l[l][7] = take(kDM);
    for (int j = 8; j < 12; ++j) o_l[l][j] = take(kDM);
  }
  const size_t o_w0 = take((size_t)kDM * kHid), o_b0 = take(kHid), o_lg = take(kHid), o_lb = take(kHid);
  const size_t o_w3 = take((size_t)kTargetDim * kHid), o_b3 = take(16);
  const size_t o_tin = take((size_t)kT * 256), o_t1 = take((size_t)kT * kTEmb), o_t2 = take((size_t)kT * kTEmb);
  DenoiserWeights* w = new (std::nothrow) DenoiserWeights();
  if (!w) { cudaFree(raw); return ctx->fail(PDB_ERR_CUDA, "out of host memory"); }
  cudaError_t err = cudaMalloc(&w->arena, sizeof(float) * total);
  if (err != cudaSuccess) { cudaFree(raw); delete w; return ctx->fail(PDB_ERR_CUDA, "weight arena: %s", cudaGetErrorString(err)); }
  w->arena_floats = total;
  float* A = w->arena;
  auto pack = [&](int ti, int O, int ldw, int c0, int Kuse, int Kpad, size_t dst) {
    const int n = (Kpad / 4) * O;
    pack_k4_kernel<<<(n + 255) / 256, 256, 0, st>>>(raw + off[ti], O, ldw, c0, Kuse, Kpad, reinterpret_cast<float4*>(A + dst));
  };
  auto copy = [&](int ti, size_t dst, size_t n) {
    cudaMemcpyAsync(A + dst, raw + off[ti], sizeof(float) * n, cudaMemcpyDeviceToDevice, st);
  };
  pack(4, kDM, kFirstIn, 0, kPoseEmb, kPoseEmbPad, o_fx);                 // harmonic pose columns
  pack(4, kDM, kFirstIn, kPoseEmb + kTEmb, kZ, kZ, o_fz);                 // z columns 317..700
  gather_col_kernel<<<(kDM + 255) / 256, 256, 0, st>>>(raw + off[4], kDM, kFirstIn, kFirstIn - 1, A + o_piv);
  copy(5, o_bf, kDM);
  for (int l = 0; l < kLayers; ++l) {
    const int b = 6 + 12 * l;
    pack(b + 0, 3 * kDM, kDM, 0, kDM, kDM, o_l[l][0]); copy(b + 1, o_l[l][1], 3 * kDM);
    pack(b + 2, kDM, kDM, 0, kDM, kDM, o_l[l][2]);     copy(b + 3, o_l[l][3], kDM);
    pack(b + 4, kFF, kDM, 0, kDM, kDM, o_l[l][4]);     copy(b + 5, o_l[l][5], kFF);
    pack(b + 6, kDM, kFF, 0, kFF, kFF, o_l[l][6]);     copy(b + 7, o_l[l][7], kDM);
    for (int j = 8; j < 12; ++j) copy(b + j, o_l[l][j], kDM);
  }
  const int tb = 6 + 12 * kLayers;
  pack(tb + 0, kHid, kDM, 0, kDM, kDM, o_w0); copy(tb + 1, o_b0, kHid);
  copy(tb + 2, o_lg, kHid); copy(tb + 3, o_lb, kHid);
  copy(tb + 4, o_w3, (size_t)kTargetDim * kHid); copy(tb + 5, o_b3, kTargetDim);
  // timestep table: [cos(t f_k) | sin(t f_k)] -> Linear(256,128) -> SiLU -> Linear(128,128) -> _first columns 189..316
  {
    std::vector<float> tin((size_t)kT * 256);
    for (int t = 0; t < kT; ++t)
      for (int k = 0; k < 128; ++k) {
        const float freq = expf(-logf(10000.0f) * (float)k / 128.0f);  // embedding.py:25 (fp32)
        const float arg = (float)t * freq;
        tin[(size_t)t * 256 + k] = cosf(arg);
        tin[(size_t)t * 256 + 128 + k] = sinf(arg);
      }
    cudaMemcpyAsync(A + o_tin, tin.data(), sizeof(float) * tin.size(), cudaMemcpyHostToDevice, st);
    cudaStreamSynchronize(st);  // tin dies at scope exit
    naive_linear_kernel<<<(kT * kTEmb + 255) / 256, 256, 0, st>>>(A + o_tin, kT, 256, raw + off[0], kTEmb, 256, 0, raw + off[1], A + o_t1, 1);
    naive_linear_kernel<<<(kT * kTEmb + 255) / 256, 256, 0, st>>>(A + o_t1, kT, kTEmb, raw + off[2], kTEmb, kTEmb, 0, raw + off[3], A + o_t2, 0);
    naive_linear_kernel<<<(kT * kDM + 255) / 256, 256, 0, st>>>(A + o_t2, kT, kTEmb, raw + off[4], kDM, kFirstIn, kPoseEmb, nullptr, A + o_tproj, 0);
  }
  {
    float sched[kT * 8];
    pdb_schedule_table(sched, 1e-4, 0.1);
    cudaMemcpyAsync(A + o_sched, sched, sizeof(sched), cudaMemcpyHostToDevice, st);
    cudaStreamSynchronize(st);
  }
  // ---- operands of the tensor-core engine: row-major weights, LayerNorm gamma/beta folded into QKV and FF1 ----
  {
    size_t tt = 0;
    auto take2 = [&](size_t n) { size_t at = tt; tt += (n + 63) / 64 * 64; return at; };
    const size_t t_wx = take2((size_t)kDM * kPoseEmbPad), t_wz = take2((size_t)kDM * kZ);
    size_t t_l[kLayers][6];
    for (int l = 0; l < kLayers; ++l) {
      t_l[l][0] = take2((size_t)3 * kDM * kDM); t_l[l][1] = take2(3 * kDM); t_l[l][2] = take2(3 * kDM);
      t_l[l][3] = take2((size_t)kFF * kDM);     t_l[l][4] = take2(kFF);     t_l[l][5] = take2(kFF);
    }
    err = cudaMalloc(&w->tc_arena, sizeof(float) * tt);
    if (err == cudaSuccess) {
      float* T = w->tc_arena;
      copy_cols_kernel<<<(kDM * kPoseEmbPad + 255) / 256, 256, 0, st>>>(raw + off[4], kDM, kFirstIn, 0, kPoseEmb, kPoseEmbPad, T + t_wx);
      copy_cols_kernel<<<(kDM * kZ + 255) / 256, 256, 0, st>>>(raw + off[4], kDM, kFirstIn, kPoseEmb + kTEmb, kZ, kZ, T + t_wz);
      TcWeights& tc = w->tc;
      tc.wx = T + t_wx; tc.wz = T + t_wz; tc.w_pivot = A + o_piv; tc.b_first = A + o_bf; tc.tproj = A + o_tproj;
      tc.wlast0 = raw + off[tb + 0]; tc.blast0 = raw + off[tb + 1];
      for (int l = 0; l < kLayers; ++l) {
        const int b = 6 + 12 * l;
        fold_ln_kernel<<<3 * kDM, 128, 0, st>>>(raw + off[b + 0], raw + off[b + 1], raw + off[b + 8], raw + off[b + 9], kDM,
                                              T + t_l[l][0], T + t_l[l][1], T + t_l[l][2]);
        fold_ln_kernel<<<kFF, 128, 0, st>>>(raw + off[b + 4], raw + off[b + 5], raw + off[b + 10], raw + off[b + 11], kDM,
                                          T + t_l[l][3], T + t_l[l][4], T + t_l[l][5]);
        TcLayer& L = tc.layer[l];
        L.wqkv = T + t_l[l][0]; L.colsum_qkv = T + t_l[l][1]; L.bias_qkv = T + t_l[l][2];
        L.wout = raw + off[b + 2]; L.bout = raw + off[b + 3];
        L.wff1 = T + t_l[l][3]; L.colsum_ff1 = T + t_l[l][4]; L.bias_ff1 = T + t_l[l][5];
        L.wff2 = raw + off[b + 6]; L.bff2 = raw + off[b + 7];
      }
    }
  }
  if (err == cudaSuccess) err = cudaStreamSynchronize(st);
  if (err == cudaSuccess) err = cudaGetLastError();
  if (err != cudaSuccess) {
    cudaFree(raw);
    if (w->tc_arena) cudaFree(w->tc_arena);
    cudaFree(w->arena);
    delete w;
    return ctx->fail(PDB_ERR_CUDA, "weight packing failed: %s", cudaGetErrorString(err));
  }
  ctx->launches += 3 + 2 + 4 * kLayers + 1 + 3;
  DenoiserDev& d = w->dev;
  d.w_first_x = reinterpret_cast<const float4*>(A + o_fx);
  d.w_first_z = reinterpret_cast<const float4*>(A + o_fz);
  d.w_first_pivot = A + o_piv;
  d.b_first = A + o_bf;
  d.tproj = A + o_tproj;
  d.sched = A + o_sched;
  for (int l = 0; l < kLayers; ++l) {
    LayerWeights& L = d.layer[l];
    L.w_qkv = reinterpret_cast<const float4*>(A + o_l[l][0]); L.b_qkv = A + o_l[l][1];
    L.w_out = reinterpret_cast<const float4*>(A + o_l[l][2]); L.b_out = A + o_l[l][3];
    L.w_ff1 = reinterpret_cast<const float4*>(A + o_l[l][4]); L.b_ff1 = A + o_l[l][5];
    L.w_ff2 = reinterpret_cast<const float4*>(A + o_l[l][6]); L.b_ff2 = A + o_l[l][7];
    L.ln1_g = A + o_l[l][8]; L.ln1_b = A + o_l[l][9]; L.ln2_g = A + o_l[l][10]; L.ln2_b = A + o_l[l][11];
  }
  d.w_last0 = reinterpret_cast<const float4*>(A + o_w0);
  d.b_last0 = A + o_b0;
  d.ln_last_g = A + o_lg;
  d.ln_last_b = A + o_lb;
  d.w_last3 = A + o_w3;
  d.b_last3 = A + o_b3;
  w->raw = raw;
  if (ctx->weights) {
    cudaFree(ctx->weights->arena);
    if (ctx->weights->raw) cudaFree(ctx->weights->raw);
    if (ctx->weights->tc_arena) cudaFree(ctx->weights->tc_arena);
    delete ctx->weights;
  }
  ctx->weights = w;
  return PDB_OK;
}

int pdb_denoiser_forward(pdb_context* c, const float* x_dev, int32_t t, const float* z_dev, int32_t batch, int32_t frames,
                         float* eps_dev, void* stream) {
  if (!c) return PDB_ERR_INVALID;
  Context* ctx = reinterpret_cast<Context*>(c);
  if (!x_dev || !z_dev || !eps_dev) return ctx->fail(PDB_ERR_INVALID, "null argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  PDB_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t n = (size_t)batch * frames * kTargetDim;
  if (int rc = ensure_buffer(ctx, &ctx->stage, &ctx->stage_bytes, sizeof(float) * n)) return rc;
  float* xs = static_cast<float*>(ctx->stage);  // the kernel advances its state in place: work on a copy
  PDB_CUDA(ctx, cudaMemcpyAsync(xs, x_dev, sizeof(float) * n, cudaMemcpyDeviceToDevice, st));
  DenoiserRun run = {};
  run.batch = batch; run.frames = frames;
  run.t_hi = run.t_lo = t;
  run.guide_below = 0;
  run.compute_zproj = 1;
  run.x = xs; run.z = z_dev;
  run.eps_out = eps_dev;
  return enqueue_denoiser(ctx, run, st);
}

int pdb_p_sample(pdb_context* c, const float* x_dev, int32_t t, const float* z_dev, const float* noise_dev, int32_t batch,
                 int32_t frames, float* pred_dev, float* mean_dev, float* x0_dev, void* stream) {
  if (!c) return PDB_ERR_INVALID;
  Context* ctx = reinterpret_cast<Context*>(c);
  if (!x_dev || !z_dev || !pred_dev) return ctx->fail(PDB_ERR_INVALID, "null argument");
  if (t < 0 || t >= kT) return ctx->fail(PDB_ERR_INVALID, "timestep %d outside [0, %d)", t, kT);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  PDB_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t n = (size_t)batch * frames * kTargetDim;
  if (pred_dev != x_dev) PDB_CUDA(ctx, cudaMemcpyAsync(pred_dev, x_dev, sizeof(float) * n, cudaMemcpyDeviceToDevice, st));
  DenoiserRun run = {};
  run.batch = batch; run.frames = frames;
  run.t_hi = run.t_lo = t;
  run.guide_below = 0;
  run.compute_zproj = 1;
  run.x = pred_dev; run.z = z_dev;
  // the kernel indexes draws as [1 + (T-1-t)]: rebase the single noise tensor accordingly
  run.draws = noise_dev ? noise_dev - (size_t)(1 + (kT - 1 - t)) * n : nullptr;
  run.mean_out = mean_dev; run.x0_out = x0_dev;
  return enqueue_denoiser(ctx, run, st);
}

int pdb_sample_loop(pdb_context* c, const float* z_dev, const float* draws_dev, int32_t batch, int32_t frames,
                    pdb_matches* const* problems, int32_t n_problems, const pdb_ggs_config* cfg, int32_t cond_start_step,
                    float* pose_dev, float* trail_dev, pdb_ggs_stats* stats_dev, void* stream) {
  if (!c) return PDB_ERR_INVALID;
  Context* ctx = reinterpret_cast<Context*>(c);
  if (!z_dev || !draws_dev || !pose_dev) return ctx->fail(PDB_ERR_INVALID, "null argument");
  if (problems && !cfg) return ctx->fail(PDB_ERR_INVALID, "GGS config missing");
  if (problems && n_problems != batch)
    return ctx->fail(PDB_ERR_INVALID, "%d match sets for a batch of %d sequences (one per sequence)", n_problems, batch);
  if (problems)  // before anything is enqueued: a set packed for another frame count would stride the pose wrongly
    if (int rc = check_ggs_problems(ctx, problems, batch, frames)) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  PDB_CUDA(ctx, cudaSetDevice(ctx->device));
  LoopState loop;
  if (int rc = loop_prefix(ctx, z_dev, draws_dev, batch, frames, problems ? cond_start_step : 0, pose_dev, trail_dev, st, &loop)) return rc;
  return loop_guided(ctx, &loop, problems, cfg, stats_dev, st);
}

int pdb_sample_loop_host(pdb_context* c, const float* z_host, const float* draws_host, int32_t batch, int32_t frames,
                         pdb_matches* const* problems, int32_t n_problems, const pdb_ggs_config* cfg, int32_t cond_start_step,
                         float* pose_host, float* trail_host, pdb_ggs_stats* stats_host, void* stream) {
  if (!c) return PDB_ERR_INVALID;
  Context* ctx = reinterpret_cast<Context*>(c);
  if (!z_host || !draws_host || !pose_host) return ctx->fail(PDB_ERR_INVALID, "null argument");
  if (problems && n_problems != batch)
    return ctx->fail(PDB_ERR_INVALID, "%d match sets for a batch of %d sequences (one per sequence)", n_problems, batch);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  PDB_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t S = (size_t)batch * frames, n = S * kTargetDim;
  const int guided = problems ? (cond_start_step < 0 ? 0 : (cond_start_step > kT ? kT : cond_start_step)) : 0;
  const size_t f_z = S * kZ, f_draws = (size_t)(kT + 1) * n, f_pose = n, f_trail = trail_host ? (size_t)(kT + 1) * n : 0;
  const size_t stats_bytes = stats_host ? sizeof(pdb_ggs_stats) * (size_t)guided * batch : 0;
  const size_t bytes = sizeof(float) * (f_z + f_draws + f_pose + f_trail) + stats_bytes + 256;
  // separate staging area from pdb_denoiser_forward's: reuse ctx->stage (grown on demand)
  if (int rc = ensure_buffer(ctx, &ctx->stage, &ctx->stage_bytes, bytes)) return rc;
  float* z_dev = static_cast<float*>(ctx->stage);
  float* draws_dev = z_dev + f_z;
  float* pose_dev = draws_dev + f_draws;
  float* trail_dev = trail_host ? pose_dev + f_pose : nullptr;
  pdb_ggs_stats* stats_dev = stats_host ? reinterpret_cast<pdb_ggs_stats*>(pose_dev + f_pose + f_trail) : nullptr;
  PDB_CUDA(ctx, cudaMemcpyAsync(z_dev, z_host, sizeof(float) * f_z, cudaMemcpyHostToDevice, st));
  PDB_CUDA(ctx, cudaMemcpyAsync(draws_dev, draws_host, sizeof(float) * f_draws, cudaMemcpyHostToDevice, st));
  if (stats_dev) PDB_CUDA(ctx, cudaMemsetAsync(stats_dev, 0, stats_bytes, st));
  if (int rc = pdb_sample_loop(c, z_dev, draws_dev, batch, frames, problems, n_problems, cfg, cond_start_step, pose_dev, trail_dev,
                               stats_dev, stream))
    return rc;
  PDB_CUDA(ctx, cudaMemcpyAsync(pose_host, pose_dev, sizeof(float) * f_pose, cudaMemcpyDeviceToHost, st));
  if (trail_host) PDB_CUDA(ctx, cudaMemcpyAsync(trail_host, trail_dev, sizeof(float) * f_trail, cudaMemcpyDeviceToHost, st));
  if (stats_host && stats_bytes) PDB_CUDA(ctx, cudaMemcpyAsync(stats_host, stats_dev, stats_bytes, cudaMemcpyDeviceToHost, st));
  PDB_CUDA(ctx, cudaStreamSynchronize(st));
  return PDB_OK;
}

// The end-to-end call of a guided run that starts from the reference's match format (host arrays, one match set per sequence):
// the match sets are packed and uploaded WHILE the unguided prefix of the loop (t = T-1 .. cond_start_step, one launch) runs on
// the GPU -- the packer is host work plus a copy on its own stream, the prefix does not need the matches.
int pdb_sample_loop_host_matches(pdb_context* c, const float* z_host, const float* draws_host, int32_t batch, int32_t frames,
                                 const double* const* kp1, const double* const* kp2, const int64_t* const* i12,
                                 const int64_t* m_total, int32_t height, int32_t width, const pdb_ggs_config* cfg,
                                 int32_t cond_start_step, float* pose_host, float* trail_host, pdb_ggs_stats* stats_host,
                                 void* stream) {
  if (!c) return PDB_ERR_INVALID;
  Context* ctx = reinterpret_cast<Context*>(c);
  if (!z_host || !draws_host || !pose_host || !kp1 || !kp2 || !i12 || !m_total || !cfg)
    return ctx->fail(PDB_ERR_INVALID, "null argument");
  if (batch < 1 || frames < 1) return ctx->fail(PDB_ERR_INVALID, "bad batch / frames");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  PDB_CUDA(ctx, cudaSetDevice(ctx->device));
  if (!ctx->pack_stream) PDB_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->pack_stream, cudaStreamNonBlocking));
  const size_t S = (size_t)batch * frames, n = S * kTargetDim;
  const int guided = cond_start_step < 0 ? 0 : (cond_start_step > kT ? kT : cond_start_step);
  const size_t f_z = S * kZ, f_draws = (size_t)(kT + 1) * n, f_pose = n, f_trail = trail_host ? (size_t)(kT + 1) * n : 0;
  const size_t stats_bytes = stats_host ? sizeof(pdb_ggs_stats) * (size_t)guided * batch : 0;
  const size_t bytes = sizeof(float) * (f_z + f_draws + f_pose + f_trail) + stats_bytes + 256;
  if (int rc = ensure_buffer(ctx, &ctx->stage, &ctx->stage_bytes, bytes)) return rc;
  float* z_dev = static_cast<float*>(ctx->stage);
  float* draws_dev = z_dev + f_z;
  float* pose_dev = draws_dev + f_draws;
  float* trail_dev = trail_host ? pose_dev + f_pose : nullptr;
  pdb_ggs_stats* stats_dev = stats_host ? reinterpret_cast<pdb_ggs_stats*>(pose_dev + f_pose + f_trail) : nullptr;
  PDB_CUDA(ctx, cudaMemcpyAsync(z_dev, z_host, sizeof(float) * f_z, cudaMemcpyHostToDevice, st));
  PDB_CUDA(ctx, cudaMemcpyAsync(draws_dev, draws_host, sizeof(float) * f_draws, cudaMemcpyHostToDevice, st));
  if (stats_dev) PDB_CUDA(ctx, cudaMemsetAsync(stats_dev, 0, stats_bytes, st));
  LoopState loop;
  if (int rc = loop_prefix(ctx, z_dev, draws_dev, batch, frames, guided, pose_dev, trail_dev, st, &loop)) return rc;
  // ---- host: pack while the prefix runs (pdb_matches_pack returns once ITS stream has taken the upload) ----
  std::vector<pdb_matches*> sets((size_t)batch, nullptr);
  int rc = PDB_OK;
  for (int b = 0; b < batch && rc == PDB_OK; ++b)
    rc = pdb_matches_pack(c, kp1[b], kp2[b], i12[b], m_total[b], frames, height, width, 0, ctx->pack_stream, &sets[b]);
  if (rc == PDB_OK) rc = check_ggs_problems(ctx, sets.data(), batch, frames);
  if (rc == PDB_OK) rc = loop_guided(ctx, &loop, sets.data(), cfg, stats_dev, st);
  cudaError_t err = cudaSuccess;
  if (rc == PDB_OK) {
    err = cudaMemcpyAsync(pose_host, pose_dev, sizeof(float) * f_pose, cudaMemcpyDeviceToHost, st);
    if (err == cudaSuccess && trail_host) err = cudaMemcpyAsync(trail_host, trail_dev, sizeof(float) * f_trail, cudaMemcpyDeviceToHost, st);
    if (err == cudaSuccess && stats_host && stats_bytes)
      err = cudaMemcpyAsync(stats_host, stats_dev, stats_bytes, cudaMemcpyDeviceToHost, st);
  }
  const cudaError_t sync = cudaStreamSynchronize(st);  // also on the error path: the match sets are released below
  for (pdb_matches* m : sets) pdb_matches_free(m);
  if (rc != PDB_OK) return rc;
  if (err != cudaSuccess || sync != cudaSuccess)
    return ctx->fail(PDB_ERR_CUDA, "sample loop failed: %s", cudaGetErrorString(err != cudaSuccess ? err : sync));
  return PDB_OK;
}

}  // extern "C"
