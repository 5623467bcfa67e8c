// TEST HARNESS (not product): runs the persistent kernels of posediffusion_b200/csrc -- the same sources nvcc compiles for
// sm_90a -- on the CPU through the execution-model emulation of cuda_emu.h: the GGS kernel body (csrc/ggs.cuh, every
// template variant and streaming mode), the fp32 denoiser kernel (csrc/denoiser.cuh) and the camera-alignment kernels
// (csrc/align.cuh).  Build:  g++ -O1 -std=c++17 -shared -fPIC (see __graft_entry__.py::build_emulator).
#include "cuda_emu.h"

#include <chrono>

#include "../../posediffusion_b200/csrc/ggs.cuh"
#include "../../posediffusion_b200/csrc/align.cuh"
#include "../../posediffusion_b200/csrc/denoiser.cuh"

// ---------------------------------------------------------------------------------------------------------------
// emulator runtime
// ---------------------------------------------------------------------------------------------------------------
namespace emu {
thread_local Cta* g_cta = nullptr;
thread_local uint3 g_threadIdx = {0, 0, 0}, g_blockIdx = {0, 0, 0};
thread_local dim3 g_blockDim(1, 1, 1), g_gridDim(1, 1, 1);

static void trampoline() {
  Cta* c = g_cta;
  const int me = c->current;
  c->body();
  c->done[me] = 1;
  c->live -= 1;
  // a finished thread no longer takes part in block barriers: release one that is now complete
  if (c->live > 0 && c->block_count == c->live) {
    c->block_count = 0;
    c->block_gen++;
  }
  swapcontext(&c->ctx[me], &c->sched);
}

static void run_cta(int block_index, int grid, int block, const std::function<void()>& body) {
  Cta cta;
  cta.nthreads = block;
  cta.nwarps = (block + kWarp - 1) / kWarp;
  cta.ctx.resize(block);
  cta.stack.resize(block);
  cta.done.assign(block, 0);
  cta.live = block;
  cta.warp_count.assign(cta.nwarps, 0);
  cta.warp_gen.assign(cta.nwarps, 0);
  cta.xch.assign((size_t)cta.nwarps * kWarp, 0);
  cta.body = body;
  cta.smem = static_cast<unsigned char*>(aligned_alloc(1024, kSharedBytes));  // the CTA's dynamic shared memory
  memset(cta.smem, 0xcd, kSharedBytes);  // shared memory is NOT zero-initialised on the device either
  g_cta = &cta;
  g_blockIdx = {(unsigned)block_index, 0, 0};
  g_blockDim = dim3(block, 1, 1);
  g_gridDim = dim3(grid, 1, 1);
  for (int t = 0; t < block; ++t) {
    cta.stack[t] = static_cast<char*>(malloc(kStackBytes));
    getcontext(&cta.ctx[t]);
    cta.ctx[t].uc_stack.ss_sp = cta.stack[t];
    cta.ctx[t].uc_stack.ss_size = kStackBytes;
    cta.ctx[t].uc_link = &cta.sched;
    makecontext(&cta.ctx[t], trampoline, 0);
  }
  // watchdog: a kernel that deadlocks (a barrier some threads never reach, an mbarrier phase that never completes) must fail
  // the test run instead of hanging it
  const char* limit_env = getenv("PDB_EMU_TIMEOUT_S");
  const double limit_s = limit_env ? atof(limit_env) : 900.0;
  const auto t_start = std::chrono::steady_clock::now();
  unsigned long passes = 0;
  while (cta.live > 0) {
    if ((++passes & 1023) == 0 && std::chrono::duration<double>(std::chrono::steady_clock::now() - t_start).count() > limit_s) {
      fprintf(stderr, "emu: CTA %d made no end after %.0f s (%d of %d threads alive, block barrier %d/%d arrived): deadlock?\n",
              block_index, limit_s, cta.live, block, cta.block_count, cta.live);
      abort();
    }
    for (int t = 0; t < block; ++t) {
      if (cta.done[t]) continue;
      cta.current = t;
      g_threadIdx = {(unsigned)t, 0, 0};
      swapcontext(&cta.sched, &cta.ctx[t]);
    }
  }
  for (int t = 0; t < block; ++t) free(cta.stack[t]);
  free(cta.smem);
  g_cta = nullptr;
}

void launch(int grid, int block, const std::function<void()>& body) {
  std::vector<std::thread> ctas;
  for (int b = 0; b < grid; ++b) ctas.emplace_back(run_cta, b, grid, block, std::cref(body));
  for (auto& t : ctas) t.join();
}
}  // namespace emu

// ---------------------------------------------------------------------------------------------------------------
// one geometry_guided_sampling / compute_sampson_distance call on the emulated grid
// ---------------------------------------------------------------------------------------------------------------
extern "C" int ggs_emu_run(const float* pts, const int* segs /*[nseg+1][4] incl. sentinel*/, int nseg, int rounds, long long m_total,
                           int frames, float height, float width, float* pose /*[frames*9] in/out*/, int paired, int eval, int cpp,
                           int force_stream, int no_ring, const int* iters, const int* flags, int n_phases, float alpha, float lr,
                           float smax, float momentum, double min_matches, float* dbg_grad, float* dbg_scalars, float* dbg_F,
                           float* dbg_G, pdb_ggs_stats* stats, int* mode_out) {
  using namespace pdb;
  if (frames < 1 || frames > kMaxFrames || cpp < 1 || n_phases < 1 || n_phases > PDB_GGS_PHASES) return -1;
  // exchange slots as api_core.cu lays them out: PDB_GGS_GROUP overrides the group size here too (tests exercise both the
  // one-level and the two-level exchange with few CTAs)
  int group = kXchGroupDefault;
  if (const char* g = getenv("PDB_GGS_GROUP")) group = atoi(g) >= 2 ? atoi(g) : 2;
  if (cpp <= 2 * group && !getenv("PDB_GGS_GROUP")) group = cpp;
  if (group >= cpp) group = cpp;
  const int groups = ggs_xch_groups(cpp, group);
  std::vector<unsigned long long> xch(2 * (size_t)(cpp + groups) * ggs_xch_words(frames), 0ull);
  GgsProblem pr = {};
  pr.pts = reinterpret_cast<const float4*>(pts);
  pr.segs = reinterpret_cast<const int4*>(segs);
  pr.nseg = nseg;
  pr.rounds = rounds;
  pr.m_total = m_total;
  pr.frames = frames;
  pr.height = height;
  pr.width = width;
  pr.pose = pose;
  pr.xch1 = xch.data();
  pr.xch2 = xch.data() + 2 * (size_t)cpp * ggs_xch_words(frames);
  std::vector<unsigned long long> acc(3 * (size_t)ggs_xch_words(frames) * kAccStride / 2 + 8, 0ull);  // 8-byte aligned accumulators
  pr.acc = reinterpret_cast<float*>(acc.data());
  pr.stats = stats;
  pr.dbg_grad = dbg_grad;
  pr.dbg_scalars = dbg_scalars;
  pr.dbg_F = dbg_F;
  pr.dbg_G = dbg_G;
  GgsParams P = {};
  P.ctas_per_problem = cpp;
  P.n_phases = n_phases;
  for (int i = 0; i < n_phases; ++i) {
    P.iters[i] = iters[i];
    P.flags[i] = flags[i];
  }
  P.alpha = alpha;
  P.lr = lr;
  P.smax = smax;
  P.momentum = momentum;
  P.min_matches = min_matches;
  P.xch_group = group;
  P.xch_mode = (getenv("PDB_GGS_XCH") && atoi(getenv("PDB_GGS_XCH")) == 0) ? 0 : 1;
  // the launch logic of api_core.cu::launch_ggs_chunk: shared-memory-resident slice when it fits, else the bulk-async ring
  const size_t fixed = ggs_smem_fixed_bytes(frames);
  const size_t budget = emu::kSharedBytes > fixed + 1024 ? emu::kSharedBytes - fixed - 1024 : 0;
  const long long rounds_per_cta = ggs_rounds_per_cta(rounds > 0 ? rounds : 1, cpp, paired != 0);
  const bool resident = (size_t)rounds_per_cta * 512 <= budget && !force_stream;
  P.resident_rounds = resident ? (int)rounds_per_cta : 0;
  P.ring = (resident || no_ring) ? 0 : 1;
  if (mode_out) *mode_out = resident ? 0 : (P.ring ? 1 : 2);
  if (fixed + (resident ? (size_t)rounds_per_cta * 512 : (size_t)kRingBytes) > emu::kSharedBytes) return -2;
  const std::function<void()> body = [&]() {
    if (eval) {
      if (paired) ggs_body<true, true>(pr, P); else ggs_body<true, false>(pr, P);
    } else {
      if (paired) ggs_body<false, true>(pr, P); else ggs_body<false, false>(pr, P);
    }
  };
  emu::launch(cpp, kGgsThreads, body);
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// camera alignment (csrc/align.cuh): the two kernel bodies with the launch geometry of pdb_cameras_align
// ---------------------------------------------------------------------------------------------------------------
extern "C" void cameras_align_emu(const float* Rs, const float* Ts, const float* Rt, const float* Tt, int count, int estimate_scale, float eps,
                                  float* Ro, float* To, float* align) {
  emu::launch(1, 32, [&]() { pdb::cameras_align_estimate_warp(Rs, Ts, Rt, Tt, count, estimate_scale, eps, align); });
  emu::launch((count + 127) / 128, 128, [&]() { pdb::cameras_align_apply_thread(align, Rs, Ts, count, Ro, To); });
}

// ---------------------------------------------------------------------------------------------------------------
// fp32 denoiser kernel (csrc/denoiser.cuh): weight re-layout as pdb_denoiser_load does it (pack_k4 / gather_col /
// naive_linear kernels of csrc/api_sampler.cu, restated as host loops), then denoiser_kernel<TS> on the emulated grid.
// tensors = the 108 checkpoint tensors in reference state_dict order (posediffusion_b200.synthetic.denoiser_param_shapes).
// ---------------------------------------------------------------------------------------------------------------
namespace {
std::vector<float> pack_k4(const float* W, int O, int ldw, int c0, int Kuse, int Kpad) {  // [O][ldw] window -> [Kpad/4][O] float4
  std::vector<float> out((size_t)Kpad * O, 0.f);
  for (int k4 = 0; k4 < Kpad / 4; ++k4)
    for (int o = 0; o < O; ++o)
      for (int j = 0; j < 4; ++j) {
        const int k = k4 * 4 + j;
        out[((size_t)k4 * O + o) * 4 + j] = (k < Kuse) ? W[(size_t)o * ldw + c0 + k] : 0.f;
      }
  return out;
}
std::vector<float> naive_linear(const float* X, int S, int K, const float* W, int O, int ldw, int c0, const float* bias, bool silu) {
  std::vector<float> Y((size_t)S * O);
  for (int s = 0; s < S; ++s)
    for (int o = 0; o < O; ++o) {
      float acc = 0.f;
      for (int k = 0; k < K; ++k) acc = fmaf(X[(size_t)s * K + k], W[(size_t)o * ldw + c0 + k], acc);
      if (bias) acc += bias[o];
      if (silu) acc = acc / (1.0f + expf(-acc));
      Y[(size_t)s * O + o] = acc;
    }
  return Y;
}
template <int TS>
void run_denoiser(const pdb::DenoiserDev& W, const pdb::DenoiserRun& R, int grid, bool flagged) {
  if (flagged) emu::launch(grid, pdb::kDenThreads, [&]() { pdb::denoiser_kernel<TS, true>(W, R); });
  else emu::launch(grid, pdb::kDenThreads, [&]() { pdb::denoiser_kernel<TS, false>(W, R); });
}
}  // namespace

extern "C" int denoiser_emu_run(const float* const* tensors, const float* sched /*[100][8]*/, int batch, int frames, int t_hi, int t_lo,
                                int guide_below, float* x /*[S,9] in/out*/, const float* z /*[S,384]*/, const float* draws /*[T+1,S,9] or null*/,
                                float* trail /*[T+1,S,9] or null*/, float* eps_out, float* x0_out, float* mean_out, int grid, int token_tile) {
  using namespace pdb;
  const int S = batch * frames;
  if (S < 1 || frames > kMaxFrames || t_hi >= kT || t_lo < 0 || t_hi < t_lo || grid < 1) return -1;
  // ---- weights: the re-layout of pdb_denoiser_load ----
  std::vector<std::vector<float>> keep;
  auto hold = [&](std::vector<float> v) { keep.push_back(std::move(v)); return keep.back().data(); };
  DenoiserDev D = {};
  D.w_first_x = reinterpret_cast<const float4*>(hold(pack_k4(tensors[4], kDM, kFirstIn, 0, kPoseEmb, kPoseEmbPad)));
  D.w_first_z = reinterpret_cast<const float4*>(hold(pack_k4(tensors[4], kDM, kFirstIn, kPoseEmb + kTEmb, kZ, kZ)));
  {
    std::vector<float> piv(kDM);
    for (int o = 0; o < kDM; ++o) piv[o] = tensors[4][(size_t)o * kFirstIn + kFirstIn - 1];
    D.w_first_pivot = hold(std::move(piv));
  }
  D.b_first = tensors[5];
  {  // timestep table (embedding.py:24-37 in fp32, as the library builds it)
    std::vector<float> tin((size_t)kT * 256);
    for (int t = 0; t < kT; ++t)
      for (int k = 0; k < 128; ++k) {
        const float freq = expf(-logf(10000.0f) * (float)k / 128.0f);
        const float arg = (float)t * freq;
        tin[(size_t)t * 256 + k] = cosf(arg);
        tin[(size_t)t * 256 + 128 + k] = sinf(arg);
      }
    std::vector<float> t1 = naive_linear(tin.data(), kT, 256, tensors[0], kTEmb, 256, 0, tensors[1], true);
    std::vector<float> t2 = naive_linear(t1.data(), kT, kTEmb, tensors[2], kTEmb, kTEmb, 0, tensors[3], false);
    D.tproj = hold(naive_linear(t2.data(), kT, kTEmb, tensors[4], kDM, kFirstIn, kPoseEmb, nullptr, false));
  }
  for (int l = 0; l < kLayers; ++l) {
    const int b = 6 + 12 * l;
    LayerWeights& L = D.layer[l];
    L.w_qkv = reinterpret_cast<const float4*>(hold(pack_k4(tensors[b + 0], 3 * kDM, kDM, 0, kDM, kDM)));
    L.b_qkv = tensors[b + 1];
    L.w_out = reinterpret_cast<const float4*>(hold(pack_k4(tensors[b + 2], kDM, kDM, 0, kDM, kDM)));
    L.b_out = tensors[b + 3];
    L.w_ff1 = reinterpret_cast<const float4*>(hold(pack_k4(tensors[b + 4], kFF, kDM, 0, kDM, kDM)));
    L.b_ff1 = tensors[b + 5];
    L.w_ff2 = reinterpret_cast<const float4*>(hold(pack_k4(tensors[b + 6], kDM, kFF, 0, kFF, kFF)));
    L.b_ff2 = tensors[b + 7];
    L.ln1_g = tensors[b + 8]; L.ln1_b = tensors[b + 9]; L.ln2_g = tensors[b + 10]; L.ln2_b = tensors[b + 11];
  }
  const int tb = 6 + 12 * kLayers;
  D.w_last0 = reinterpret_cast<const float4*>(hold(pack_k4(tensors[tb + 0], kHid, kDM, 0, kDM, kDM)));
  D.b_last0 = tensors[tb + 1];
  D.ln_last_g = tensors[tb + 2];
  D.ln_last_b = tensors[tb + 3];
  D.w_last3 = tensors[tb + 4];
  D.b_last3 = tensors[tb + 5];
  D.sched = sched;
  // ---- run descriptor + workspace (enqueue_denoiser of csrc/api_sampler.cu) ----
  std::vector<float> ws(denoiser_ws_floats(S) + 64, 0.f);
  DenoiserRun R = {};
  R.batch = batch; R.frames = frames; R.tokens = S;
  R.t_hi = t_hi; R.t_lo = t_lo; R.guide_below = guide_below; R.compute_zproj = 1;
  R.x = x; R.z = z; R.draws = draws; R.trail = trail; R.eps_out = eps_out; R.x0_out = x0_out; R.mean_out = mean_out;
  float* p = ws.data();
  R.bar = reinterpret_cast<unsigned*>(p); p += 64;
  R.zproj = p; p += (size_t)S * kDM;
  R.h = p;     p += (size_t)S * kDM;
  R.qkv = p;   p += (size_t)S * 3 * kDM;
  R.att = p;   p += (size_t)S * kDM;
  R.ff = p;    p += (size_t)S * kFF;
  R.u = p;
  // stage hand-over as enqueue_denoiser selects it: flag-carrying words when PDB_DEN_FLAG=1.  The buffers start out holding
  // stale words of an "earlier launch" (tags below tag_base, garbage values) so that a reader that accepts a wrong version fails.
  const bool flagged = getenv("PDB_DEN_FLAG") && atoi(getenv("PDB_DEN_FLAG")) != 0;
  std::vector<unsigned long long> fws(denoiser_flag_ws_words(S) + 16);
  const unsigned tag_base = 1000u;
  for (size_t i = 0; i < fws.size(); ++i) fws[i] = ((unsigned long long)(tag_base - 1u - (unsigned)(i % 7)) << 32) | 0x7fc00000ull;  // NaN payloads
  {
    unsigned long long* fw = fws.data();
    R.fh = fw;   fw += (size_t)S * kDM;
    R.fqkv = fw; fw += (size_t)S * 2 * 3 * kDM;
    R.fatt = fw; fw += (size_t)S * kDM;
    R.fff = fw;  fw += (size_t)S * kFF;
    R.fu = fw;   fw += (size_t)S * kHid;
    R.fx = fw;
    R.tag_base = tag_base;
  }
  if (denoiser_smem_bytes(token_tile, frames) > emu::kSharedBytes) return -2;
  switch (token_tile) {
    case 8: run_denoiser<8>(D, R, grid, flagged); break;
    case 16: run_denoiser<16>(D, R, grid, flagged); break;
    case 20: run_denoiser<20>(D, R, grid, flagged); break;
    case 24: run_denoiser<24>(D, R, grid, flagged); break;
    case 32: run_denoiser<32>(D, R, grid, flagged); break;
    default: return -3;
  }
  return 0;
}
