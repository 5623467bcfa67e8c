// TEST HARNESS (not product): one geometry_guided_sampling call on the emulated grid (cuda_emu.h) with either the reproducible
// instantiation of ggs_body (csrc/ggs.cuh, kRepro, as pdb_set_reproducible launches it) or the default one, under a chosen
// schedule.  Linked into build/libkernels_emu.so next to kernels_emu.cpp, which provides the emulator runtime (emu::launch).
//
// Scheduling knob: the emulator resumes the coroutines of a CTA in index order, a warp at a time.  This file gives coroutine warp
// w the kernel's warp perm(w) -- schedule 0: w (the emulator's own order), 1: nwarps - 1 - w (reversed), k >= 2: (w + k) % nwarps
// (rotated) -- by reading threadIdx through the permutation.  Lanes keep their index, so the emulator's warp collectives still
// pair the right threads; only the order in which the kernel's warps reach each shared-memory or global sum changes.  The
// kernel source is compiled here in a namespace of its own (pdb -> pdb_sched), so that its instantiations with the permuted
// threadIdx never meet the ones of kernels_emu.cpp at link time.
#include "cuda_emu.h"

namespace ggs_sched {
int g_schedule = 0;
inline uint3 thread_index() {
  const int c = emu::g_cta->current, nw = emu::g_cta->nwarps, w = c / emu::kWarp;
  const int kw = g_schedule == 1 ? nw - 1 - w : g_schedule >= 2 ? (w + g_schedule) % nw : w;
  return make_uint3((unsigned)(kw * emu::kWarp + c % emu::kWarp), 0u, 0u);
}
}  // namespace ggs_sched

#undef threadIdx
#define threadIdx (ggs_sched::thread_index())
#define pdb pdb_sched
#include "../../posediffusion_b200/csrc/ggs.cuh"
#undef pdb

// Arguments as ggs_emu_run (kernels_emu.cpp), optimisation only (five phases); repro = 1: the reproducible instantiation with the
// slot exchange, 0: the default instantiation with the exchange PDB_GGS_XCH selects.  Returns -1 for bad arguments, -2 when the
// shared memory does not fit.
extern "C" int ggs_emu_run_scheduled(const float* pts, const int* segs /*[nseg+1][4] incl. sentinel*/, int nseg, int rounds,
                                     long long m_total, int frames, float height, float width, float* pose /*[frames*9] in/out*/,
                                     int paired, int cpp, int force_stream, int no_ring, const int* iters, const int* flags, int n_phases,
                                     float alpha, float lr, float smax, float momentum, double min_matches, pdb_ggs_stats* stats,
                                     int* mode_out, int repro, int schedule) {
  using namespace pdb_sched;
  if (frames < 1 || frames > kMaxFrames || cpp < 1 || n_phases < 1 || n_phases > PDB_GGS_PHASES || schedule < 0) return -1;
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
  P.xch_mode = (repro || (getenv("PDB_GGS_XCH") && atoi(getenv("PDB_GGS_XCH")) == 0)) ? 0 : 1;  // as enqueue_ggs
  // the launch logic of api_core.cu::launch_ggs_chunk: resident slice when it fits, else the bulk-async ring
  const size_t fixed = ggs_smem_fixed_bytes(frames, repro != 0);
  const size_t budget = emu::kSharedBytes > fixed + 1024 ? emu::kSharedBytes - fixed - 1024 : 0;
  const long long rounds_per_cta = ggs_rounds_per_cta(rounds > 0 ? rounds : 1, cpp, paired != 0);
  const bool resident = (size_t)rounds_per_cta * 512 <= budget && !force_stream;
  P.resident_rounds = resident ? (int)rounds_per_cta : 0;
  P.ring = (resident || no_ring) ? 0 : 1;
  if (mode_out) *mode_out = resident ? 0 : (P.ring ? 1 : 2);
  if (fixed + (resident ? (size_t)rounds_per_cta * 512 : (size_t)kRingBytes) > emu::kSharedBytes) return -2;
  const std::function<void()> body = [&]() {
    if (repro) {
      if (paired) ggs_body<false, true, false, false, true>(pr, P); else ggs_body<false, false, false, false, true>(pr, P);
    } else {
      if (paired) ggs_body<false, true>(pr, P); else ggs_body<false, false>(pr, P);
    }
  };
  ggs_sched::g_schedule = schedule;
  emu::launch(cpp, kGgsThreads, body);
  ggs_sched::g_schedule = 0;
  return 0;
}
