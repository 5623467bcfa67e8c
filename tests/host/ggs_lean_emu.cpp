// TEST HARNESS (not product): one geometry_guided_sampling call on the emulated grid (cuda_emu.h) with the instantiation the
// library's launch would pick -- the lean ggs_body (csrc/ggs.cuh, kLean) when the slice is resident, every CTA touches at
// most kGgsMaxSeg segments (ggs_lean_fits), the exchange is the one-hop mode and the call optimises, else the general one.
// Linked into build/libkernels_emu.so next to kernels_emu.cpp, which provides the emulator runtime (emu::launch).
#include "cuda_emu.h"

#include "../../posediffusion_b200/csrc/ggs.cuh"

// Same arguments as ggs_emu_run (kernels_emu.cpp); *lean_out = 1 when the lean instantiation ran.
extern "C" int ggs_emu_run_dispatch(const float* pts, const int* segs /*[nseg+1][4] incl. sentinel*/, int nseg, int rounds,
                                    long long m_total, int frames, float height, float width, float* pose /*[frames*9] in/out*/,
                                    int paired, int eval, int cpp, int force_stream, int no_ring, const int* iters, const int* flags,
                                    int n_phases, float alpha, float lr, float smax, float momentum, double min_matches,
                                    float* dbg_grad, float* dbg_scalars, float* dbg_F, float* dbg_G, pdb_ggs_stats* stats,
                                    int* mode_out, int* lean_out) {
  using namespace pdb;
  if (frames < 1 || frames > kMaxFrames || cpp < 1 || n_phases < 1 || n_phases > PDB_GGS_PHASES) return -1;
  // exchange workspace as api_core.cu lays it out (PDB_GGS_GROUP overrides the group size as in ggs_emu_run)
  int group = kXchGroupDefault;
  if (const char* g = getenv("PDB_GGS_GROUP")) group = atoi(g) >= 2 ? atoi(g) : 2;
  if (cpp <= 2 * group && !getenv("PDB_GGS_GROUP")) group = cpp;
  if (group >= cpp) group = cpp;
  const int groups = ggs_xch_groups(cpp, group);
  std::vector<unsigned long long> xch(2 * (size_t)(cpp + groups) * ggs_xch_words(frames), 0ull);
  std::vector<unsigned long long> acc(3 * (size_t)ggs_xch_words(frames) * kAccStride / 2 + 8, 0ull);  // 8-byte aligned accumulators
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
  // the launch logic of api_core.cu::launch_ggs_chunk: resident slice when it fits, else the bulk-async ring; then the lean rule
  const size_t fixed = ggs_smem_fixed_bytes(frames);
  const size_t budget = emu::kSharedBytes > fixed + 1024 ? emu::kSharedBytes - fixed - 1024 : 0;
  const long long rounds_per_cta = ggs_rounds_per_cta(rounds > 0 ? rounds : 1, cpp, paired != 0);
  const bool resident = (size_t)rounds_per_cta * 512 <= budget && !force_stream;
  P.resident_rounds = resident ? (int)rounds_per_cta : 0;
  P.ring = (resident || no_ring) ? 0 : 1;
  const bool lean = !eval && resident && P.xch_mode == 1 && ggs_lean_fits(pr.segs, nseg, rounds, cpp, paired != 0);
  if (mode_out) *mode_out = resident ? 0 : (P.ring ? 1 : 2);
  if (lean_out) *lean_out = lean ? 1 : 0;
  if (fixed + (resident ? (size_t)rounds_per_cta * 512 : (size_t)kRingBytes) > emu::kSharedBytes) return -2;
  const std::function<void()> body = [&]() {
    if (eval) {
      if (paired) ggs_body<true, true>(pr, P); else ggs_body<true, false>(pr, P);
    } else if (lean) {
      if (paired) ggs_body<false, true, false, true>(pr, P); else ggs_body<false, false, false, true>(pr, P);
    } else {
      if (paired) ggs_body<false, true>(pr, P); else ggs_body<false, false>(pr, P);
    }
  };
  emu::launch(cpp, kGgsThreads, body);
  return 0;
}
