// C-ABI entry points: denoiser weights, denoiser forward, p_sample, p_sample_loop (device and host buffers), and its DDIM forms
// (a strided prefix, and optionally guided DDIM jumps; DESIGN.md "Fewer-step sampling").
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

int enqueue_denoiser_tc(Context* ctx, const DenoiserDev& dev, DenoiserRun run, cudaStream_t st);
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
int launch_denoiser(Context* ctx, const DenoiserDev& dev, const DenoiserRun& run, int grid, cudaStream_t st) {
  const size_t smem = denoiser_smem_bytes(TS, run.frames);
  if (smem > ctx->smem_optin) return ctx->fail(PDB_ERR_LIMIT, "denoiser needs %zu B shared memory", smem);
  size_t& attr_bytes = ctx->attr->den[(kFlag ? 8 : 0) + TS / 4 - 1];  // static shared memory counts against the opt-in limit: ask for what we use
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
    PDB_CUDA(ctx, cudaLaunchKernelEx(&cfg, denoiser_kernel<TS, kFlag>, dev, run));
  }
  ctx->launches += 1;
  return PDB_OK;
}

// Fill the workspace pointers of `run` and launch steps t_hi..t_lo.  `tables` (may be NULL: the loaded weights' own) is a copy of
// the weight descriptor whose per-timestep rows -- `tproj` and `sched` -- are those of a DDIM step table (make_ddim_tables).
int enqueue_denoiser(Context* ctx, DenoiserRun run, cudaStream_t st, const DenoiserDev* tables = nullptr) {
  if (!ctx->weights) return ctx->fail(PDB_ERR_STATE, "denoiser weights not loaded (pdb_denoiser_load)");
  const DenoiserDev& dev = tables ? *tables : ctx->weights->dev;
  if (run.batch < 1 || run.frames < 1) return ctx->fail(PDB_ERR_INVALID, "empty batch");
  if (run.frames > PDB_MAX_FRAMES) return ctx->fail(PDB_ERR_LIMIT, "frames %d > PDB_MAX_FRAMES", run.frames);
  if (run.t_hi >= kT || run.t_lo < 0 || run.t_hi < run.t_lo) return ctx->fail(PDB_ERR_INVALID, "bad timestep range");
  const int S = run.batch * run.frames;
  run.tokens = S;
  // engine: exact-fp32 persistent kernel below kTcMinTokens tokens (latency bound), wgmma/TMA tiles (TF32 products) at or
  // above it (throughput bound).  ctx->denoiser_engine: 0 auto, 1 force fp32, 2 force tensor cores.
  const bool use_tc = ctx->denoiser_engine == 2 || (ctx->denoiser_engine == 0 && S >= kTcMinTokens);
  if (use_tc) return enqueue_denoiser_tc(ctx, dev, run, st);
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
      case 8: return launch_denoiser<8, true>(ctx, dev, run, grid, st);
      case 16: return launch_denoiser<16, true>(ctx, dev, run, grid, st);
      case 20: return launch_denoiser<20, true>(ctx, dev, run, grid, st);
      case 24: return launch_denoiser<24, true>(ctx, dev, run, grid, st);
      default: return launch_denoiser<32, true>(ctx, dev, run, grid, st);
    }
  }
  switch (TS) {
    case 8: return launch_denoiser<8, false>(ctx, dev, run, grid, st);
    case 16: return launch_denoiser<16, false>(ctx, dev, run, grid, st);
    case 20: return launch_denoiser<20, false>(ctx, dev, run, grid, st);
    case 24: return launch_denoiser<24, false>(ctx, dev, run, grid, st);
    default: return launch_denoiser<32, false>(ctx, dev, run, grid, st);
  }
}

// float64 betas (torch.linspace: filled symmetrically from both ends) and their cumulative product
void schedule_f64(double beta_1, double beta_T, double* beta, double* abar) {
  const int n = kT;
  const double step = (beta_T - beta_1) / (double)(n - 1);
  for (int i = 0; i < n; ++i) beta[i] = (i < n / 2) ? beta_1 + step * i : beta_T - step * (n - 1 - i);
  double prod = 1.0;
  for (int i = 0; i < n; ++i) {
    prod *= (1.0 - beta[i]);
    abar[i] = prod;
  }
}

// Guided jump times tau'_j = floor(j g / g') - 1, j = 0 .. g': tau'_{g'} = g - 1 (where the prefix lands), tau'_0 = -1 (x0).
int guided_time(int j, int g, int gs) { return (int)((long long)j * g / gs) - 1; }

// DDIM step table (Song et al. 2021, eq. 12; DESIGN.md "Fewer-step sampling").  Entries 0 .. k-1 (k = steps - guided_steps) jump
// tau_{k-i} -> tau_{k-i-1}, tau_j = (g - 1) + floor(j (T - g) / k), abar(-1) = 1.  Entries k .. steps-1 are the guided tail: with
// guided_steps == g the DDPM rows of timesteps g-1 .. 0, else g' DDIM jumps tau'_{g'-i} -> tau'_{g'-i-1} at the same eta.  False
// for g' outside [min(1, g), g], k outside [1, T - g], eta < 0 or not finite, or an eta > 1 so large that 1 - abar_s - sigma^2 < 0
// at some jump.
bool ddim_table(int steps, int guide_below, int guided_steps, double eta, double beta_1, double beta_T, int32_t* t_out,
                float* coef_out) {
  const int g = guide_below, gs = guided_steps, k = steps - guided_steps;
  if (g < 0 || g > kT || gs < (g > 0 ? 1 : 0) || gs > g || k < 1 || k > kT - g || !std::isfinite(eta) || eta < 0.0) return false;
  double beta[kT], abar[kT];
  schedule_f64(beta_1, beta_T, beta, abar);
  auto jump = [&](int t, int s, int i) {
    const double at = abar[t], as = s < 0 ? 1.0 : abar[s];
    const double sigma = eta * std::sqrt((1.0 - as) / (1.0 - at)) * std::sqrt(1.0 - at / as);
    const double rest = 1.0 - as - sigma * sigma;
    if (!(rest >= 0.0)) return false;
    const double c2 = std::sqrt(rest) / std::sqrt(1.0 - at);
    const double c1 = std::sqrt(as) - c2 * std::sqrt(at);
    float* r = coef_out + i * 8;
    r[0] = (float)std::sqrt(1.0 / at);  // a_t, b_t exactly as the schedule rows hold them
    r[1] = (float)std::sqrt(1.0 / at - 1.0);
    r[2] = (float)c1;
    r[3] = (float)c2;
    r[4] = (float)sigma;
    r[5] = (float)s;
    r[6] = (float)at;
    r[7] = (float)as;
    t_out[i] = t;
    return true;
  };
  for (int i = 0; i < k; ++i) {
    const int j = k - i;
    if (!jump((g - 1) + (int)((long long)j * (kT - g) / k), (g - 1) + (int)((long long)(j - 1) * (kT - g) / k), i)) return false;
  }
  if (gs < g) {
    for (int i = 0; i < gs; ++i)
      if (!jump(guided_time(gs - i, g, gs), guided_time(gs - i - 1, g, gs), k + i)) return false;
    return true;
  }
  float sched[kT * 8];
  pdb_schedule_table(sched, beta_1, beta_T);
  for (int i = 0; i < g; ++i) {
    t_out[k + i] = g - 1 - i;
    std::memcpy(coef_out + (size_t)(k + i) * 8, sched + (size_t)(g - 1 - i) * 8, sizeof(float) * 8);
  }
  return true;
}

// dst[v_i] = src[t_i] (512 floats): the time-embedding block of step i's real timestep at its virtual timestep
struct RowMap { int dst[kT]; int src[kT]; };
__global__ void gather_tproj_kernel(const float* __restrict__ src, float* __restrict__ dst, RowMap map) {
  const int i = blockIdx.x;
  for (int c = threadIdx.x; c < kDM; c += blockDim.x) dst[(size_t)map.dst[i] * kDM + c] = src[(size_t)map.src[i] * kDM + c];
}

// A DDIM loop as the kernels see it: a copy of the weight descriptor whose per-timestep tables are indexed by virtual timesteps --
// sched[v] = a step's DDIM coefficient row, tproj[v] = the time-embedding block of its real timestep.  Prefix step i sits at
// v = T-1-i, so the DDPM loop over v = T-1 .. T-k IS the DDIM prefix, draw and trail slot 1 + i included.  The `jumps` guided
// jumps (table entries k ..; 0 when the tail stays DDPM) sit at v = jumps-1 .. 0: below guide_below, so the kernel adds no noise
// and writes no trail slot for them; jumps <= g <= T - k keeps the two ranges apart.  The tables live in a context-owned buffer at
// a fixed address, rewritten (stream-ordered) before each loop.
int make_ddim_tables(Context* ctx, const int32_t* tab_t, const float* tab_coef, int k, int jumps, cudaStream_t st, DenoiserDev* out) {
  const size_t sched_floats = (size_t)kT * 8, bytes = sizeof(float) * (sched_floats + (size_t)kT * kDM);
  if (!ctx->step_tab) PDB_CUDA(ctx, cudaMalloc(&ctx->step_tab, bytes));
  float* vsched = static_cast<float*>(ctx->step_tab);
  float* vtproj = vsched + sched_floats;
  float rows[kT * 8] = {};
  RowMap map = {};
  for (int i = 0; i < k + jumps; ++i) {
    const int v = i < k ? kT - 1 - i : k + jumps - 1 - i;
    std::memcpy(rows + (size_t)v * 8, tab_coef + (size_t)i * 8, sizeof(float) * 8);
    map.dst[i] = v;
    map.src[i] = tab_t[i];
  }
  PDB_CUDA(ctx, cudaMemcpyAsync(vsched, rows, sizeof(rows), cudaMemcpyHostToDevice, st));
  *out = ctx->weights->dev;
  gather_tproj_kernel<<<k + jumps, 128, 0, st>>>(out->tproj, vtproj, map);
  PDB_CUDA(ctx, cudaGetLastError());
  ctx->launches += 1;
  out->tproj = vtproj;
  out->sched = vsched;
  return PDB_OK;
}

int clamp_guided(int cond_start_step) { return cond_start_step < 0 ? 0 : (cond_start_step > kT ? kT : cond_start_step); }

// The match sets of a host-matches entry: the reference's host arrays, one sequence each, packed while the prefix runs.
struct HostMatches {
  const double* const* kp1;
  const double* const* kp2;
  const int64_t* const* i12;
  const int64_t* m_total;
  int height, width;
};

// One call of a sampling-loop entry point.  z / draws / pose / trail / stats are device buffers, or host buffers that host_loop
// stages.  Match sets come packed (`problems`), as host arrays (`pack`), or not at all.
struct LoopArgs {
  const float* z;
  const float* draws;
  int batch, frames;
  pdb_matches* const* problems;
  int n_problems;
  const HostMatches* pack;
  const pdb_ggs_config* cfg;
  int cond_start_step;
  float* pose;
  float* trail;
  pdb_ggs_stats* stats;
  bool ddim = false;  // the loop of pdb_sample_loop_ddim_guided: `steps` evaluations, the last `guided_steps` the guided tail
  int steps = 0;
  double eta = 0.0;
  int guided_steps = 0;
};

// The loop as the kernels run it, built and checked by plan_loop before anything is enqueued.  The prefix is ONE launch over
// timesteps T-1 .. T-prefix_steps: the DDPM steps t = T-1 .. g, or the k DDIM steps at virtual timesteps T-1 .. T-k of the step
// tables (make_ddim_tables).  The tail takes tail_steps denoiser steps at timesteps tail_steps-1 .. 0, each followed by GGS in
// place and a copy into trail slot 1 + prefix_steps + i: the g DDPM steps on the weights' own tables (also after a DDIM prefix:
// the tensor-core engine keys its captured step graph on the table addresses), or g' < g DDIM jumps on the step tables (below
// guide_below, so the kernel leaves the mean, adds no noise and writes no trail slot).  Not copyable: the descriptors may point
// at steps_dev.
struct LoopPlan {
  LoopPlan() = default;
  LoopPlan(const LoopPlan&) = delete;
  int g = 0;                 // guide_below: clamp(cond_start_step, 0, T); 0 for a DDPM loop without match sets
  int prefix_steps = 0;      // T - g (DDPM, none at g = T) or k (DDIM)
  int tail_steps = 0;        // g (DDPM) or g' (DDIM) with match sets, else 0
  const DenoiserDev* prefix_tables = nullptr;
  const DenoiserDev* tail_tables = nullptr;
  bool noise = true;         // the kernel adds noise from draws[1 + i] (false: DDIM at eta = 0, whose draws are x_T alone)
  size_t draw_slots = 0, trail_slots = 0, stats_rows = 0;
  bool ddim = false;         // DDIM: the step table's rows, its prefix steps k and guided jumps (0: a DDPM tail)
  int jumps = 0;
  int32_t t[kT];
  float coef[kT * 8];
  DenoiserDev steps_dev;     // the step tables, filled by run_loop
};

// Every check of a sampling-loop call, made before anything is enqueued.  Only a match set that fails to pack is found later,
// while the prefix runs (run_loop).
int plan_loop(Context* ctx, const LoopArgs& a, LoopPlan* p) {
  const HostMatches* hm = a.pack;
  if (!a.z || !a.draws || !a.pose || (hm && (!hm->kp1 || !hm->kp2 || !hm->i12 || !hm->m_total || !a.cfg)))
    return ctx->fail(PDB_ERR_INVALID, "null argument");
  if (a.batch < 1 || a.frames < 1) return ctx->fail(PDB_ERR_INVALID, "empty batch");
  if (a.frames > PDB_MAX_FRAMES) return ctx->fail(PDB_ERR_LIMIT, "frames %d > PDB_MAX_FRAMES", a.frames);
  if (!ctx->weights) return ctx->fail(PDB_ERR_STATE, "denoiser weights not loaded (pdb_denoiser_load)");
  const bool sets = a.problems || hm;
  if (sets && !a.cfg) return ctx->fail(PDB_ERR_INVALID, "GGS config missing");
  if (a.problems) {
    if (a.n_problems != a.batch)
      return ctx->fail(PDB_ERR_INVALID, "%d match sets for a batch of %d sequences (one per sequence)", a.n_problems, a.batch);
    // a set packed for another frame count would stride the pose wrongly
    if (int rc = check_ggs_problems(ctx, a.problems, a.batch, a.frames)) return rc;
  }
  p->g = sets || a.ddim ? clamp_guided(a.cond_start_step) : 0;
  p->prefix_tables = p->tail_tables = &ctx->weights->dev;
  p->ddim = a.ddim;
  if (a.ddim) {
    if (!ddim_table(a.steps, p->g, a.guided_steps, a.eta, 1e-4, 0.1, p->t, p->coef))
      return ctx->fail(PDB_ERR_INVALID,
                       "DDIM: %d denoiser steps, %d of them over %d guided timesteps (the guided tail needs %d .. %d, the unguided "
                       "prefix 1 .. %d) and eta %g (>= 0, finite)",
                       a.steps, a.guided_steps, p->g, p->g > 0 ? 1 : 0, p->g, kT - p->g, a.eta);
    p->prefix_steps = a.steps - a.guided_steps;
    p->jumps = a.guided_steps < p->g ? a.guided_steps : 0;
    p->tail_steps = sets ? a.guided_steps : 0;  // without match sets the prefix alone runs: pose = x_{g-1}
    p->prefix_tables = &p->steps_dev;
    if (p->jumps) p->tail_tables = &p->steps_dev;
    p->noise = a.eta > 0.0;
    p->draw_slots = p->noise ? 1 + p->prefix_steps : 1;
    p->trail_slots = 1 + a.steps;
  } else {
    p->prefix_steps = kT - p->g;
    p->tail_steps = p->g;
    p->draw_slots = p->trail_slots = kT + 1;
  }
  p->stats_rows = p->tail_steps;
  if (p->tail_steps && a.cfg->iter_num < 0) return ctx->fail(PDB_ERR_INVALID, "iter_num < 0");
  return PDB_OK;
}

// The sampling loop of every entry point, on device buffers: fill the step tables (DDIM), enqueue x_T = draws[0]
// (gaussian_diffuser.py:289) and the prefix, take the match sets -- given, or packed into `packed` now, while the prefix runs (the
// caller frees them once the stream is synchronised) -- and enqueue the guided tail.
int run_loop(Context* ctx, const LoopArgs& a, LoopPlan* p, cudaStream_t st, std::vector<pdb_matches*>* packed) {
  if (p->ddim)
    if (int rc = make_ddim_tables(ctx, p->t, p->coef, p->prefix_steps, p->jumps, st, &p->steps_dev)) return rc;
  const size_t n = (size_t)a.batch * a.frames * kTargetDim;
  PDB_CUDA(ctx, cudaMemcpyAsync(a.pose, a.draws, sizeof(float) * n, cudaMemcpyDeviceToDevice, st));
  if (a.trail) PDB_CUDA(ctx, cudaMemcpyAsync(a.trail, a.draws, sizeof(float) * n, cudaMemcpyDeviceToDevice, st));
  DenoiserRun run = {};
  run.batch = a.batch; run.frames = a.frames;
  run.guide_below = p->g;
  run.x = a.pose; run.z = a.z; run.draws = p->noise ? a.draws : nullptr; run.trail = a.trail;
  run.compute_zproj = 1;
  if (p->prefix_steps > 0) {
    run.t_hi = kT - 1; run.t_lo = kT - p->prefix_steps;
    if (int rc = enqueue_denoiser(ctx, run, st, p->prefix_tables)) return rc;
    run.compute_zproj = 0;
  }
  pdb_matches* const* sets = a.problems;
  if (const HostMatches* hm = a.pack) {  // pdb_matches_pack returns once ITS stream has taken the upload
    if (!ctx->pack_stream) PDB_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->pack_stream, cudaStreamNonBlocking));
    packed->assign((size_t)a.batch, nullptr);
    for (int b = 0; b < a.batch; ++b)
      if (int rc = pdb_matches_pack(reinterpret_cast<pdb_context*>(ctx), hm->kp1[b], hm->kp2[b], hm->i12[b], hm->m_total[b], a.frames,
                                    hm->height, hm->width, 0, ctx->pack_stream, &(*packed)[b]))
        return rc;
    sets = packed->data();
    if (int rc = check_ggs_problems(ctx, sets, a.batch, a.frames)) return rc;
  }
  for (int i = 0; i < p->tail_steps; ++i) {
    run.t_hi = run.t_lo = p->tail_steps - 1 - i;
    if (int rc = enqueue_denoiser(ctx, run, st, p->tail_tables)) return rc;
    run.compute_zproj = 0;
    pdb_ggs_stats* stats = a.stats ? a.stats + (size_t)i * a.batch : nullptr;
    if (int rc = enqueue_ggs(ctx, sets, a.batch, a.frames, a.pose, a.cfg, stats, st)) return rc;
    if (a.trail)
      PDB_CUDA(ctx, cudaMemcpyAsync(a.trail + (size_t)(1 + p->prefix_steps + i) * n, a.pose, sizeof(float) * n,
                                    cudaMemcpyDeviceToDevice, st));
  }
  return PDB_OK;
}

int device_loop(pdb_context* c, const LoopArgs& a, void* stream) {
  if (!c) return PDB_ERR_INVALID;
  Context* ctx = reinterpret_cast<Context*>(c);
  LoopPlan plan;
  if (int rc = plan_loop(ctx, a, &plan)) return rc;
  PDB_CUDA(ctx, cudaSetDevice(ctx->device));
  return run_loop(ctx, a, &plan, static_cast<cudaStream_t>(stream), nullptr);
}

// The host-buffer entries: one staging buffer ctx->stage = [z | draws | pose | trail | stats] laid out from the plan's slot counts
// (separate from pdb_denoiser_forward's use of it, grown on demand), z and the draws copied in, the loop, then pose, trail and
// stats copied out and the stream synchronised -- on the error path too, before packed match sets are released.
int host_loop(pdb_context* c, const LoopArgs& h, void* stream) {
  if (!c) return PDB_ERR_INVALID;
  Context* ctx = reinterpret_cast<Context*>(c);
  LoopPlan plan;
  if (int rc = plan_loop(ctx, h, &plan)) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  PDB_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t n = (size_t)h.batch * h.frames * kTargetDim;
  const size_t f_z = (size_t)h.batch * h.frames * kZ, f_draws = plan.draw_slots * n, f_trail = h.trail ? plan.trail_slots * n : 0;
  const size_t stats_bytes = h.stats ? sizeof(pdb_ggs_stats) * plan.stats_rows * h.batch : 0;
  if (int rc = ensure_buffer(ctx, &ctx->stage, &ctx->stage_bytes, sizeof(float) * (f_z + f_draws + n + f_trail) + stats_bytes + 256))
    return rc;
  float* z = static_cast<float*>(ctx->stage);
  float* draws = z + f_z;
  float* pose = draws + f_draws;
  LoopArgs d = h;
  d.z = z; d.draws = draws; d.pose = pose;
  d.trail = h.trail ? pose + n : nullptr;
  d.stats = h.stats ? reinterpret_cast<pdb_ggs_stats*>(pose + n + f_trail) : nullptr;
  PDB_CUDA(ctx, cudaMemcpyAsync(z, h.z, sizeof(float) * f_z, cudaMemcpyHostToDevice, st));
  PDB_CUDA(ctx, cudaMemcpyAsync(draws, h.draws, sizeof(float) * f_draws, cudaMemcpyHostToDevice, st));
  if (d.stats) PDB_CUDA(ctx, cudaMemsetAsync(d.stats, 0, stats_bytes, st));
  std::vector<pdb_matches*> packed;
  const int rc = run_loop(ctx, d, &plan, st, &packed);
  cudaError_t err = cudaSuccess;
  if (rc == PDB_OK) {
    err = cudaMemcpyAsync(h.pose, pose, sizeof(float) * n, cudaMemcpyDeviceToHost, st);
    if (err == cudaSuccess && h.trail) err = cudaMemcpyAsync(h.trail, d.trail, sizeof(float) * f_trail, cudaMemcpyDeviceToHost, st);
    if (err == cudaSuccess && h.stats && stats_bytes) err = cudaMemcpyAsync(h.stats, d.stats, stats_bytes, cudaMemcpyDeviceToHost, st);
  }
  const cudaError_t sync = cudaStreamSynchronize(st);
  for (pdb_matches* m : packed) pdb_matches_free(m);
  if (rc != PDB_OK) return rc;
  if (err != cudaSuccess || sync != cudaSuccess)
    return ctx->fail(PDB_ERR_CUDA, "sample loop failed: %s", cudaGetErrorString(err != cudaSuccess ? err : sync));
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
  if (ctx->step_tab) cudaFree(ctx->step_tab);
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
  schedule_f64(beta_1, beta_T, beta, abar);
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
  return device_loop(c, {z_dev, draws_dev, batch, frames, problems, n_problems, nullptr, cfg, cond_start_step, pose_dev, trail_dev,
                         stats_dev}, stream);
}

int pdb_ddim_table(int32_t steps, int32_t guide_below, double eta, double beta_1, double beta_T, int32_t* t_out, float* coef_out) {
  return pdb_ddim_table_guided(steps, guide_below, guide_below, eta, beta_1, beta_T, t_out, coef_out);
}

int pdb_ddim_table_guided(int32_t steps, int32_t guide_below, int32_t guided_steps, double eta, double beta_1, double beta_T,
                          int32_t* t_out, float* coef_out) {
  if (!t_out || !coef_out) return PDB_ERR_INVALID;
  return ddim_table(steps, guide_below, guided_steps, eta, beta_1, beta_T, t_out, coef_out) ? PDB_OK : PDB_ERR_INVALID;
}

int pdb_sample_loop_ddim(pdb_context* c, const float* z_dev, const float* draws_dev, int32_t batch, int32_t frames, int32_t steps,
                         double eta, pdb_matches* const* problems, int32_t n_problems, const pdb_ggs_config* cfg, int32_t cond_start_step,
                         float* pose_dev, float* trail_dev, pdb_ggs_stats* stats_dev, void* stream) {
  return pdb_sample_loop_ddim_guided(c, z_dev, draws_dev, batch, frames, steps, eta, clamp_guided(cond_start_step), problems,
                                     n_problems, cfg, cond_start_step, pose_dev, trail_dev, stats_dev, stream);
}

int pdb_sample_loop_ddim_guided(pdb_context* c, const float* z_dev, const float* draws_dev, int32_t batch, int32_t frames,
                                int32_t steps, double eta, int32_t guided_steps, pdb_matches* const* problems, int32_t n_problems,
                                const pdb_ggs_config* cfg, int32_t cond_start_step, float* pose_dev, float* trail_dev,
                                pdb_ggs_stats* stats_dev, void* stream) {
  return device_loop(c, {z_dev, draws_dev, batch, frames, problems, n_problems, nullptr, cfg, cond_start_step, pose_dev, trail_dev,
                         stats_dev, true, steps, eta, guided_steps}, stream);
}

int pdb_sample_loop_host(pdb_context* c, const float* z_host, const float* draws_host, int32_t batch, int32_t frames,
                         pdb_matches* const* problems, int32_t n_problems, const pdb_ggs_config* cfg, int32_t cond_start_step,
                         float* pose_host, float* trail_host, pdb_ggs_stats* stats_host, void* stream) {
  return host_loop(c, {z_host, draws_host, batch, frames, problems, n_problems, nullptr, cfg, cond_start_step, pose_host, trail_host,
                       stats_host}, stream);
}

// The end-to-end call of a guided run that starts from the reference's match format (host arrays, one match set per sequence):
// the match sets are packed and uploaded WHILE the unguided prefix of the loop runs on the GPU -- the packer is host work plus a
// copy on its own stream, the prefix does not need the matches.
int pdb_sample_loop_host_matches(pdb_context* c, const float* z_host, const float* draws_host, int32_t batch, int32_t frames,
                                 const double* const* kp1, const double* const* kp2, const int64_t* const* i12,
                                 const int64_t* m_total, int32_t height, int32_t width, const pdb_ggs_config* cfg,
                                 int32_t cond_start_step, float* pose_host, float* trail_host, pdb_ggs_stats* stats_host,
                                 void* stream) {
  const HostMatches hm = {kp1, kp2, i12, m_total, height, width};
  return host_loop(c, {z_host, draws_host, batch, frames, nullptr, batch, &hm, cfg, cond_start_step, pose_host, trail_host,
                       stats_host}, stream);
}

int pdb_sample_loop_host_matches_ddim(pdb_context* c, const float* z_host, const float* draws_host, int32_t batch, int32_t frames,
                                      int32_t steps, double eta, int32_t guided_steps, const double* const* kp1,
                                      const double* const* kp2, const int64_t* const* i12, const int64_t* m_total, int32_t height,
                                      int32_t width, const pdb_ggs_config* cfg, int32_t cond_start_step, float* pose_host,
                                      float* trail_host, pdb_ggs_stats* stats_host, void* stream) {
  const HostMatches hm = {kp1, kp2, i12, m_total, height, width};
  return host_loop(c, {z_host, draws_host, batch, frames, nullptr, batch, &hm, cfg, cond_start_step, pose_host, trail_host,
                       stats_host, true, steps, eta, guided_steps}, stream);
}

}  // extern "C"
