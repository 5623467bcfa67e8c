// Geometry-guided sampling on the device: one persistent cooperative kernel runs ALL phases and ALL
// SGD iterations of one `geometry_guided_sampling` call (util/geometry_guided_sampling.py:14-126) for a
// batch of independent sequences, with no host round trip.
//
// Per inner iteration (reference: one compute_sampson_distance forward + autograd backward + clip + SGD step):
//   stage 0  every CTA turns the pose (kept in shared memory, identical in all CTAs of the group) into per-frame
//            terms: R_cv, A = hat(t) R_cv, the shared mean focal length, and the K-folded At = K^-T A, Rt = K^-T R;
//   stage 1  each warp streams its contiguous slice of the packed matches (16 B per match, coalesced float4,
//            kGgsUnroll rounds in flight); F' of the current pair is 9 lanes x 6 FMAs + shuffles; the error
//            statistics and the 3x3 gradient G = sum d err / d F' accumulate in registers, then one 16-shuffle
//            warp reduction and shared-memory adds per (warp, pair segment);
//   stage 2a one warp per pair segment applies the pair adjoint on 18 lanes (G -> gAt, gRt of both frames);
//   stage 2b one thread per frame unfolds K and applies the frame adjoint (-> gT, gq): the CTA's partial gradient,
//            7 floats per frame + 4 scalars + the valid count, in shared memory;
//   exchange all-reduce of that vector over the CTAs of the sequence through L2 with flag-carrying 64-bit words
//            (common.cuh st_ll / ll_sum): every CTA publishes its vector into its own slot; with more than
//            `xch_group` CTAs the leader of each group of `xch_group` CTAs sums its group's slots (fixed order) and
//            publishes a group slot, and every CTA sums the group slots (fixed order).  No atomics, no barrier
//            counter, no accumulator to recycle; all CTAs obtain bit-identical sums; slots are double-buffered by the
//            iteration parity (a CTA can only be one exchange ahead of the slowest reader of its slot);
//   stage 3  every CTA redundantly finishes the step from the summed gradient: early-exit test, gradient mask,
//            norm-relative clip (each warp reduces the norms itself: no block barrier), momentum, update of its own
//            copy of the pose into the second pose buffer, then stage 0 of the next iteration.
#pragma once
#include "geom.cuh"
#include "ggs_layout.cuh"
#include "posediff_b200.h"

namespace pdb {

constexpr int kGgsThreads = 512;
constexpr int kGgsWarps = kGgsThreads / 32;
constexpr int kGgsMaxSeg = 128;   // pair segments handled per chunk by one CTA
constexpr int kGgsUnroll = 4;     // rounds (of 32 matches) per streaming chunk (2 KB)
constexpr int kRingStages = 4;    // chunks in flight per warp in the bulk-async ring (8 KB per warp, 128 KB per CTA)
constexpr int kRingBytes = kGgsWarps * kRingStages * kGgsUnroll * 512 + kGgsWarps * kRingStages * 8;
constexpr int kAccTail = 5;       // {g_fx', g_fy', clamp_sum, valid error sum (eval mode), valid count (int32 bits)}
constexpr int kSegAcc = 12;       // per-segment shared accumulators: G[9], clamp_sum, valid error sum, pad
constexpr int kXchGroupDefault = 12;  // CTAs per exchange group (two-level all-reduce above this many CTAs per sequence)

struct GgsProblem {
  const float4* pts;    // [rounds*32] (u1,v1,u2,v2), padded per segment to 32-row rounds
  const int4* segs;     // [nseg+1] {first_round, count, frame_a, frame_b}; sentinel {rounds,0,0,0}
  int nseg;
  int rounds;
  long long m_total;
  int frames;
  float height, width;
  float* pose;          // [frames*9] in/out
  unsigned long long* xch1;  // [2][ctas_per_problem][frames*7 + kAccTail] exchange slots of the CTAs, zero on entry
  unsigned long long* xch2;  // [2][groups][frames*7 + kAccTail] exchange slots of the group leaders, zero on entry
  float* acc;                // one-hop exchange: [3][frames*7 + kAccTail][kAccStride] {sum, arrivals} accumulators, zero on entry
  pdb_ggs_stats* stats; // may be null
  float* dbg_grad;      // eval mode: [frames*9]
  float* dbg_scalars;   // eval mode: [4]
  float* dbg_F;         // eval mode, may be null: [nseg*9]
  float* dbg_G;         // eval mode, may be null: [nseg*9], zero on entry
  long long* dbg_clock; // may be null: [ctas][8] per-stage cycle sums (stage timing probe)
};

struct GgsParams {
  int ctas_per_problem;
  int n_phases;
  int iters[PDB_GGS_PHASES];
  int flags[PDB_GGS_PHASES];  // bit0 R, bit1 T, bit2 FL
  float alpha, lr, smax, momentum;
  double min_matches;
  int resident_rounds;  // rounds of 32 matches that fit the CTA's shared-memory match cache (0 = always stream)
  int ring;             // 1: shared memory holds the bulk-async streaming ring (used when the slice is not resident)
  int xch_group;        // CTAs per exchange group; >= ctas_per_problem: one-level exchange (every CTA reads every slot)
  int xch_mode;         // 0: flag-carrying words through slots (xch1 / xch2); 1: one hop through vector reductions (acc)
};
constexpr int kAccStride = 32;  // floats between two accumulators: one 128-byte line each (one CTA per SM adding into neighbouring
                                // sectors serialise on a few L2 slices: 3.4 us per all-reduce at 32 B, 2.2 us at 128 B, tools/xchg_probe.cu)

__host__ __device__ inline int ggs_xch_words(int frames) { return frames * 7 + kAccTail; }
__host__ __device__ inline int ggs_xch_groups(int cpp, int group) { return group >= cpp ? 0 : (cpp + group - 1) / group; }

constexpr int kGgsFixedFloatsPerFrame = 2 * 9 + 4 * 9 + 4 + 18 + 14;  // pose, vel, R, A, Rt, At, fl, inr, gAt|gRt, partial + summed gradient

__host__ __device__ inline size_t ggs_smem_fixed_bytes(int frames) {
  size_t bytes = sizeof(float) * ((size_t)frames * kGgsFixedFloatsPerFrame + 128 + (size_t)kGgsMaxSeg * kSegAcc);
  bytes += kGgsMaxSeg * sizeof(int);         // segment valid counts
  bytes += 2 * (size_t)frames * sizeof(int);  // exchange plan: contributors per frame, own frames
  bytes += (kGgsMaxSeg + 1) * sizeof(int4);  // segment descriptors
  return (bytes + 127) / 128 * 128;
}

// Element-wise float2 arithmetic, one match per component.  Correctly rounded FMA / multiply / add: __fmul_rn and __fadd_rn are
// never contracted into an FMA, so every component is rounded exactly as the formula is written.
#ifdef PDB_EMU
inline float2 fma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
inline float2 mul2(float2 a, float2 b) { return make_float2(a.x * b.x, a.y * b.y); }
inline float2 add2(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
#else
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 add2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
#endif
// Two matches per call: two independent dependency chains interleaved, which keeps the FMA pipe busy in stage 1.  Same
// formulas as `sampson_match` (geom.cuh) for two in-bounds rows A and B of the same pair; acc2[k] holds separate partial
// sums for the two rows (merged at the segment end).
__device__ __forceinline__ void sampson_match2_core(const float2 u1, const float2 v1, const float2 u2, const float2 v2,
                                                    const float* __restrict__ F, float smax, float2* __restrict__ acc2) {
  float2 F2[9];  // (F'[k], F'[k])
#pragma unroll
  for (int k = 0; k < 9; ++k) F2[k] = make_float2(F[k], F[k]);
  const float2 l0 = fma2(u1, F2[0], fma2(v1, F2[3], F2[6]));
  const float2 l1 = fma2(u1, F2[1], fma2(v1, F2[4], F2[7]));
  const float2 l2 = fma2(u1, F2[2], fma2(v1, F2[5], F2[8]));
  const float2 r0 = fma2(F2[0], u2, fma2(F2[1], v2, F2[2]));
  const float2 r1 = fma2(F2[3], u2, fma2(F2[4], v2, F2[5]));
  const float2 top = fma2(l0, u2, fma2(l1, v2, l2));
  const float2 bottom = fma2(l0, l0, fma2(l1, l1, fma2(r0, r0, mul2(r1, r1))));
  const float2 t = mul2(top, make_float2(fast_rcp(bottom.x), fast_rcp(bottom.y)));
  const float2 err = mul2(top, t);
  const float2 wgt = make_float2(err.x < smax ? 1.f : 0.f, err.y < smax ? 1.f : 0.f);
  const float2 a = mul2(wgt, add2(t, t));
  const float2 nb = mul2(a, make_float2(-t.x, -t.y));
  acc2[9] = add2(acc2[9], make_float2(err.x > smax ? smax : err.x, err.y > smax ? smax : err.y));
  acc2[11] = add2(acc2[11], wgt);
  const float2 w0 = fma2(a, u2, mul2(nb, l0)), w1 = fma2(a, v2, mul2(nb, l1));
  const float2 c0 = mul2(nb, r0), c1 = mul2(nb, r1);
  acc2[0] = fma2(c0, u2, fma2(u1, w0, acc2[0]));
  acc2[1] = fma2(c0, v2, fma2(u1, w1, acc2[1]));
  acc2[2] = add2(fma2(u1, a, acc2[2]), c0);
  acc2[3] = fma2(c1, u2, fma2(v1, w0, acc2[3]));
  acc2[4] = fma2(c1, v2, fma2(v1, w1, acc2[4]));
  acc2[5] = add2(fma2(v1, a, acc2[5]), c1);
  acc2[6] = add2(acc2[6], w0);
  acc2[7] = add2(acc2[7], w1);
  acc2[8] = add2(acc2[8], a);
}
// plain layout: the rows of two rounds, one float4 (u1,v1,u2,v2) each -> the compiler re-pairs the components (MOVs)
__device__ __forceinline__ void sampson_match2(const float4 A, const float4 B, const float* __restrict__ F, float smax,
                                               float2* __restrict__ acc2) {
  sampson_match2_core(make_float2(A.x, B.x), make_float2(A.y, B.y), make_float2(A.z, B.z), make_float2(A.w, B.w), F, smax, acc2);
}
// paired layout (ggs_layout.cuh): X = (u1_A,u1_B,v1_A,v1_B), Y = (u2_A,u2_B,v2_A,v2_B) are already the operand pairs
__device__ __forceinline__ void sampson_match2_unit(const float4 X, const float4 Y, const float* __restrict__ F, float smax,
                                                    float2* __restrict__ acc2) {
  sampson_match2_core(make_float2(X.x, X.y), make_float2(X.z, X.w), make_float2(Y.x, Y.y), make_float2(Y.z, Y.w), F, smax, acc2);
}

// All-reduce of one CTA's partial gradient vector over the `cpp` CTAs of its sequence (see the file header).  Word layout:
// [0, 7N) gT | gq per frame, then g_fx', g_fy', clamp_sum, valid error sum (eval mode), valid count (int32).  On return
// s_gsum holds the sums -- the same bits in every CTA -- once the caller has passed a block barrier.  Kept out of line: its
// 16-loads-in-flight polling loops would otherwise compete for registers with the streaming loop of stage 1.
template <bool kEval>
__device__ __noinline__ void ggs_exchange(unsigned long long* xch1, unsigned long long* xch2, float* accbase, int cpp, int cta, int group,
                                          int N, unsigned it_global, const float* s_part, const float* s_misc, int cta_cnt, float g_fx,
                                          float g_fy, float* s_gsum, const int* s_expect, const int* s_mine) {
  const int tid = threadIdx.x;
  const int nsum = ggs_xch_words(N);
  if (accbase) {
    // ONE hop: a CTA adds {value, 1} to the accumulators of the frames its segments touch (s_mine; zeros if the gradient of a
    // touched frame happens to vanish) and to the five scalars; an accumulator of frame n expects s_expect[n] arrivals, a scalar
    // `cpp`.  The valid count travels as a packed 64-bit integer {arrivals : count}.  Everybody polls until the arrivals are complete.  Three buffers rotate; CTA 0 clears the one used by the previous iteration -- every CTA
    // has read it (they all contributed to this iteration afterwards) and nobody adds to it before two more exchanges.
    float* acc = accbase + (size_t)(it_global % 3u) * nsum * kAccStride;
    for (int e = tid; e < nsum; e += kGgsThreads) {
      float* slot = acc + (size_t)e * kAccStride;
      if (e < N * 7) {
        if (s_mine[e / 7]) red_pair_add(slot, s_part[e]);
      } else if (e == N * 7 + 0) red_pair_add(slot, g_fx);
      else if (e == N * 7 + 1) red_pair_add(slot, g_fy);
      else if (e == N * 7 + 2) red_pair_add(slot, s_misc[4]);
      else if (e == N * 7 + 3) red_pair_add(slot, kEval ? s_misc[5] : 0.f);
      else red_add_u64(reinterpret_cast<unsigned long long*>(slot), (1ull << 32) | (unsigned long long)(unsigned)cta_cnt);
    }
    for (int e = tid; e < nsum; e += kGgsThreads) {
      const float* slot = acc + (size_t)e * kAccStride;
      if (e < nsum - 1) {
        const float want = (float)(e < N * 7 ? s_expect[e / 7] : cpp);
        float2 v;
        for (;;) {
          v = ld_pair(slot);
          if (v.y == want) break;
          ll_backoff();
        }
        s_gsum[e] = v.x;
      } else {
        unsigned long long w;
        for (;;) {
          w = ld_ll(reinterpret_cast<const unsigned long long*>(slot));
          if ((unsigned)(w >> 32) == (unsigned)cpp) break;
          ll_backoff();
        }
        s_gsum[e] = __uint_as_float((unsigned)w);
      }
    }
    if (cta == 0) {
      float* old = accbase + (size_t)((it_global + 2u) % 3u) * nsum * kAccStride;
      for (int e = tid; e < nsum; e += kGgsThreads) st_pair_zero(old + (size_t)e * kAccStride);
      fence_gpu();  // the zeros are in place before this CTA's next contribution can be observed
    }
    return;
  }
  const unsigned tag = it_global + 1u;
  const size_t buf = it_global & 1u;
  unsigned long long* mine = xch1 + (buf * (size_t)cpp + (size_t)cta) * nsum;
  for (int e = tid; e < nsum; e += kGgsThreads) {
    unsigned bits;
    if (e < N * 7) bits = __float_as_uint(s_part[e]);
    else if (e == N * 7 + 0) bits = __float_as_uint(g_fx);
    else if (e == N * 7 + 1) bits = __float_as_uint(g_fy);
    else if (e == N * 7 + 2) bits = __float_as_uint(s_misc[4]);
    else if (e == N * 7 + 3) bits = __float_as_uint(kEval ? s_misc[5] : 0.f);
    else bits = (unsigned)cta_cnt;
    st_ll(mine + e, bits, tag);
  }
  const int groups = ggs_xch_groups(cpp, group);
  if (groups > 0) {
    const int g = cta / group;
    if (cta - g * group == 0) {  // group leader: sum the slots of the group in CTA order, publish the group slot
      const int c_lo = g * group, c_n = min(cpp, c_lo + group) - c_lo;
      const unsigned long long* src = xch1 + (buf * (size_t)cpp + (size_t)c_lo) * nsum;
      unsigned long long* dst = xch2 + (buf * (size_t)groups + (size_t)g) * nsum;
      for (int e = tid; e < nsum; e += kGgsThreads)
        st_ll(dst + e, e == nsum - 1 ? ll_sum<true>(src + e, nsum, c_n, tag) : ll_sum<false>(src + e, nsum, c_n, tag), tag);
    }
    const unsigned long long* src = xch2 + buf * (size_t)groups * nsum;
    for (int e = tid; e < nsum; e += kGgsThreads)
      s_gsum[e] = __uint_as_float(e == nsum - 1 ? ll_sum<true>(src + e, nsum, groups, tag) : ll_sum<false>(src + e, nsum, groups, tag));
  } else {
    const unsigned long long* src = xch1 + buf * (size_t)cpp * nsum;
    for (int e = tid; e < nsum; e += kGgsThreads)
      s_gsum[e] = __uint_as_float(e == nsum - 1 ? ll_sum<true>(src + e, nsum, cpp, tag) : ll_sum<false>(src + e, nsum, cpp, tag));
  }
}

// One CTA of the group that owns one sequence.  See the file header for the stage structure.
// `resident_rounds` > 0: the CTA's whole slice of matches (<= resident_rounds rounds) is staged in shared memory
// once per launch and every inner iteration streams it from there (no L2/HBM traffic inside the loop).
// kProbe: the stage timing probe (tools/ggs_stage_probe.py) is a separate instantiation, so that the production kernels carry no
// clock reads: the code one iteration executes is close to the capacity of the instruction cache.
template <bool kEval, bool kPaired = false, bool kProbe = false>
__device__ __forceinline__ void ggs_body(const GgsProblem& pr, const GgsParams& P) {
#ifdef PDB_EMU  // tests/host/cuda_emu.h (CPU emulation of this kernel, test harness only): dynamic shared memory of this CTA
  unsigned char* const smem_raw = emu::g_cta->smem;
#else
  extern __shared__ __align__(128) unsigned char smem_raw[];
#endif
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int cpp = P.ctas_per_problem;
  const int cta = blockIdx.x % cpp;
  const int N = pr.frames, N9 = N * 9;
  const int nsum = ggs_xch_words(N);

  // ---- shared memory carve-up ----
  int4* s_seg = reinterpret_cast<int4*>(smem_raw);
  float* s_pose = reinterpret_cast<float*>(s_seg + kGgsMaxSeg + 1);
  float* s_vel = s_pose + N9;
  float* s_R = s_vel + N9;
  float* s_A = s_R + N9;
  float* s_Rt = s_A + N9;
  float* s_At = s_Rt + N9;
  float* s_fl = s_At + N9;          // clamped focal lengths [N][2]
  float* s_inr = s_fl + 2 * N;      // 1 where the clamp passes gradient
  float* s_fg = s_inr + 2 * N;      // [N][18]: gAt (0..8), gRt (9..17)
  float* s_misc = s_fg + 2 * N9;    // [4] clamp_sum, [5] loss_sum, [8..11] sum over frames of d/d(ix, iy, kx, ky), [16..47] norm partials
  float* s_part = s_misc + 64;      // [N*7] this CTA's partial gradient of the iteration
  float* s_gsum = s_part + N * 7 + 32;  // [N*7 + kAccTail] summed gradient of this iteration (all CTAs: identical bits)
  float* s_sacc = s_gsum + N * 7 + 32;  // [kGgsMaxSeg][kSegAcc]
  int* s_scnt = reinterpret_cast<int*>(s_sacc + kGgsMaxSeg * kSegAcc);
  int* s_expect = s_scnt + kGgsMaxSeg;  // [N] CTAs of this sequence that contribute to frame n (one-hop exchange)
  int* s_mine = s_expect + N;           // [N] 1 if this CTA's segments touch frame n
  float4* s_pts = reinterpret_cast<float4*>(smem_raw + ggs_smem_fixed_bytes(N));
  __shared__ int s_cta_cnt;

  // ---- static work partition: rounds -> CTAs -> warps ----
  const long long R = pr.rounds;
  int r_cta0, r_cta1, r_w0, r_w1;  // paired layout: all four are even (whole units of two rounds)
  ggs_cta_range(R, cta, cpp, kPaired, &r_cta0, &r_cta1);
  auto seg_of_round = [&](int r) {  // last segment whose first_round <= r
    int lo = 0, hi = pr.nseg;       // segs[nseg].x == rounds > r
    while (hi - lo > 1) {
      int mid = (lo + hi) >> 1;
      if (__ldg(&pr.segs[mid].x) <= r) lo = mid; else hi = mid;
    }
    return lo;
  };
  const bool cta_has_work = r_cta1 > r_cta0;
  const int seg_lo = cta_has_work ? seg_of_round(r_cta0) : 0;
  const int seg_hi = cta_has_work ? seg_of_round(r_cta1 - 1) : -1;  // inclusive
  ggs_warp_range_seg(pr.segs, seg_lo, seg_hi, r_cta0, r_cta1, warp, kGgsWarps, kPaired, &r_w0, &r_w1);  // no warp crosses a segment
  const int wseg0 = (r_w1 > r_w0) ? seg_of_round(r_w0) : 0;
  const bool single_chunk = (seg_hi - seg_lo + 1) <= kGgsMaxSeg;
  const bool resident = (r_cta1 - r_cta0) <= P.resident_rounds;
  const bool use_ring = !resident && single_chunk && P.ring;
  // bulk-async ring of this warp: kRingStages chunks of kGgsUnroll rounds + one mbarrier per stage
  const uint32_t ring_base = smem_u32(s_pts) + warp * (kRingStages * kGgsUnroll * 512);
  const uint32_t ring_bar = smem_u32(s_pts) + kGgsWarps * kRingStages * kGgsUnroll * 512 + warp * (kRingStages * 8);
  const float4* ring_ptr = s_pts + warp * (kRingStages * kGgsUnroll * 32);
  unsigned ring_phase = 0;  // bit s = parity to wait for on stage s (warp-uniform, persists across iterations)
  if (use_ring && lane == 0) {
    for (int st = 0; st < kRingStages; ++st) mbar_init(ring_bar + st * 8, 1);
    mbar_fence_init();
  }

  for (int e = tid; e < N9; e += kGgsThreads) {
    s_pose[e] = pr.pose[e];
    s_vel[e] = 0.f;
  }
  for (int e = tid; e < 2 * N9; e += kGgsThreads) s_fg[e] = 0.f;
  for (int e = tid; e < kGgsMaxSeg * kSegAcc; e += kGgsThreads) s_sacc[e] = 0.f;
  for (int e = tid; e < kGgsMaxSeg; e += kGgsThreads) s_scnt[e] = 0;
  if (tid < 64) s_misc[tid] = 0.f;
  if (tid == 0) s_cta_cnt = 0;
  if (single_chunk && cta_has_work && tid <= seg_hi - seg_lo + 1) s_seg[tid] = __ldg(&pr.segs[seg_lo + tid]);
  if (resident) {
    const float4* src = pr.pts + (size_t)r_cta0 * 32;
    const int count = (r_cta1 - r_cta0) * 32;
    for (int e = tid; e < count; e += kGgsThreads) s_pts[e] = ld_stream_f4(src + e);
  }
  // ---- exchange plan (static): a CTA only adds to the accumulators of the frames its pair segments touch, and every CTA knows
  // how many contributions each frame's accumulators will receive (thread c replays the partition of CTA c)
  for (int e = tid; e < 2 * N; e += kGgsThreads) s_expect[e] = 0;  // s_expect and s_mine are adjacent
  __syncthreads();
  for (int c = tid; c < cpp; c += kGgsThreads) {
    int a0, a1;
    ggs_cta_range(R, c, cpp, kPaired, &a0, &a1);
    if (a1 > a0) {
      const int lo = seg_of_round(a0), hi = seg_of_round(a1 - 1);
      unsigned long long m_lo = 0ull, m_hi = 0ull;  // kMaxFrames = 128 frame bits
      for (int sg = lo; sg <= hi; ++sg) {
        const int4 d = __ldg(&pr.segs[sg]);
        if (d.z < 64) m_lo |= 1ull << d.z; else m_hi |= 1ull << (d.z - 64);
        if (d.w < 64) m_lo |= 1ull << d.w; else m_hi |= 1ull << (d.w - 64);
      }
      for (int n = 0; n < N; ++n) {
        const bool on = (n < 64 ? (m_lo >> n) : (m_hi >> (n - 64))) & 1ull;
        if (on) {
          atomicAdd(&s_expect[n], 1);
          if (c == cta) s_mine[n] = 1;
        }
      }
    }
  }
  static_assert(kMaxFrames <= 128, "frame bit masks of the exchange plan");
  const float scale = 0.5f * fminf(pr.height, pr.width);
  const float cx = 0.5f * pr.width, cy = 0.5f * pr.height;
  // per-launch constants of the step (the divisions are off the per-iteration dependency chain)
  const float scale_over_N = scale / (float)N, inv_m_total = 1.0f / (float)pr.m_total, alpha_over_lr = P.alpha / P.lr;
  unsigned it_global = 0;
  float kin[4] = {0.f, 0.f, 0.f, 0.f}, fpx = 1.f, fpy = 1.f;  // shared intrinsics (every warp holds a copy)

  // Pose -> per-frame terms, three threads per frame: thread (n, j < 3) builds column j of R_cv, A = hat(t) R_cv and of the
  // K-folded At, Rt.  The clamped focal lengths of the current pose are already in s_fl / s_inr (written with the pose), so
  // one block barrier suffices; every warp ends up with the shared intrinsics in registers.
  auto focal_of = [&](float log_f, float* fl, float* inr) {
    const float ev = expf(log_f + kLogFlBias);
    *fl = fminf(fmaxf(ev, kFlMin), kFlMax);
    *inr = (ev >= kFlMin && ev <= kFlMax) ? 1.f : 0.f;
  };
  auto frames_forward = [&]() {
    {  // shared focal length = mean over frames (geometry_guided_sampling.py:142), reduced redundantly per warp
      float fx = 0.f, fy = 0.f;
      for (int m = lane; m < N; m += 32) {
        fx += s_fl[m * 2];
        fy += s_fl[m * 2 + 1];
      }
      fpx = warp_sum(fx) * scale_over_N;
      fpy = warp_sum(fy) * scale_over_N;
      kin[0] = 1.f / fpx;
      kin[1] = 1.f / fpy;
      kin[2] = -cx * kin[0];
      kin[3] = -cy * kin[1];
    }
    const int n = tid >> 2, j = tid & 3;
    if (n < N && j < 3) {
      const float* p = s_pose + n * 9;
      const float w = p[3], x = p[4], y = p[5], z = p[6];
      const float s2 = 2.0f / (w * w + x * x + y * y + z * z);
      // row j of the pytorch3d rotation = column j of R_cv up to the signs D = diag(-1,-1,1) on the rows
      float r0, r1, r2;
      if (j == 0) { r0 = 1.f - s2 * (y * y + z * z); r1 = s2 * (x * y - z * w); r2 = s2 * (x * z + y * w); }
      else if (j == 1) { r0 = s2 * (x * y + z * w); r1 = 1.f - s2 * (x * x + z * z); r2 = s2 * (y * z - x * w); }
      else { r0 = s2 * (x * z - y * w); r1 = s2 * (y * z + x * w); r2 = 1.f - s2 * (x * x + y * y); }
      const float Rc[3] = {-r0, -r1, r2};
      const float tx = -p[0], ty = -p[1], tz = p[2];
      const float Ac[3] = {-tz * Rc[1] + ty * Rc[2], tz * Rc[0] - tx * Rc[2], -ty * Rc[0] + tx * Rc[1]};
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        s_R[n * 9 + i * 3 + j] = Rc[i];
        s_A[n * 9 + i * 3 + j] = Ac[i];
      }
      s_At[n * 9 + 0 + j] = kin[0] * Ac[0];
      s_At[n * 9 + 3 + j] = kin[1] * Ac[1];
      s_At[n * 9 + 6 + j] = kin[2] * Ac[0] + kin[3] * Ac[1] + Ac[2];
      s_Rt[n * 9 + 0 + j] = kin[0] * Rc[0];
      s_Rt[n * 9 + 3 + j] = kin[1] * Rc[1];
      s_Rt[n * 9 + 6 + j] = kin[2] * Rc[0] + kin[3] * Rc[1] + Rc[2];
    }
    __syncthreads();
  };
  static_assert(4 * kMaxFrames <= kGgsThreads, "four threads per frame");
  __syncthreads();
  if (tid < 2 * N) focal_of(s_pose[(tid >> 1) * 9 + 7 + (tid & 1)], &s_fl[tid], &s_inr[tid]);
  __syncthreads();
  frames_forward();

  __shared__ long long clk_sum[8];  // probe (thread 0): {stage 3 norms, stage 1, stage 2b, exchange, stage 2a, iterations, next stage 0, stage 3 update}
  if (tid < 8) clk_sum[tid] = 0;
  for (int phase = 0; phase < P.n_phases; ++phase) {
    const int flags = P.flags[phase];
    const bool upd_R = flags & 1, upd_T = flags & 2, upd_FL = flags & 4;
    const int iters = P.iters[phase];
    int done = 0, dropped = 0, last_valid = 0;          // tracked by warp 0
    float last_logged = __int_as_float(0x7fc00000);
    for (int iter = 0; iter < iters; ++iter) {
      long long ck0 = 0, ck1 = 0, ck2 = 0, ck3 = 0, ck1a = 0;  // stage timing probe (thread 0; the sums are flushed once per launch)
      if (kProbe && pr.dbg_clock && tid == 0) ck0 = clock64();
      // ================= chunks of <= kGgsMaxSeg pair segments (one chunk in all practical cases) =================
      for (int cs = seg_lo; cs <= seg_hi; cs += kGgsMaxSeg) {
        const int ce = min(cs + kGgsMaxSeg, seg_hi + 1);
        const int nchunk = ce - cs;
        if (!single_chunk) {
          __syncthreads();
          if (tid <= nchunk) s_seg[tid] = __ldg(&pr.segs[cs + tid]);
          __syncthreads();
        }
        // ---- stage 1: stream the matches of this warp's rounds ----
        {
          if (use_ring) {
            const int nr_w = r_w1 - r_w0;
            if (nr_w > 0) {
              const int nch = (nr_w + kGgsUnroll - 1) / kGgsUnroll;
              auto issue = [&](int c) {  // lane 0: request chunk c into stage c % kRingStages
                const int st = c % kRingStages;
                const int rounds_c = min(kGgsUnroll, nr_w - c * kGgsUnroll);
                mbar_arrive_expect_tx(ring_bar + st * 8, rounds_c * 512);
                bulk_copy_g2s_hint(ring_base + st * (kGgsUnroll * 512), pr.pts + (size_t)(r_w0 + c * kGgsUnroll) * 32, rounds_c * 512,
                                   ring_bar + st * 8, l2_policy_evict_first());  // the stream must not evict the exchange accumulators from L2
              };
              if (lane == 0)
                for (int c = 0; c < min(kRingStages, nch); ++c) issue(c);
              int s = wseg0;
              int4 sd = s_seg[s - cs];
              int seg_end = s_seg[s - cs + 1].x;
              float Fm[9], g[16];
              float2 g2[12];  // non-eval kernel: the accumulators live here (x = scalar path and row A, y = row B)
              int nval = 0;
              auto begin_segment = [&]() {
                float mine = 0.f;
                if (lane < 9 && sd.z != sd.w)
                  mine = pair_F_entry(s_At + sd.z * 9, s_Rt + sd.z * 9, s_At + sd.w * 9, s_Rt + sd.w * 9, lane / 3, lane % 3);
#pragma unroll
                for (int k = 0; k < 9; ++k) Fm[k] = __shfl_sync(0xffffffffu, mine, k);
                if (kEval && pr.dbg_F && lane < 9) pr.dbg_F[(size_t)s * 9 + lane] = mine;
                if (kEval) {
#pragma unroll
                  for (int k = 0; k < 16; ++k) g[k] = 0.f;
                } else {
#pragma unroll
                  for (int k = 0; k < 12; ++k) g2[k] = make_float2(0.f, 0.f);
                }
                nval = 0;
              };
              auto end_segment = [&]() {
                if (!kEval) {
#pragma unroll
                  for (int k = 0; k < 12; ++k) g[k] = g2[k].x + g2[k].y;
#pragma unroll
                  for (int k = 12; k < 16; ++k) g[k] = 0.f;
                }
                nval = __reduce_add_sync(0xffffffffu, (int)g[11]);  // per-lane counts are exact small integers
                const float tot = warp_reduce16(g, lane);
                const int slot = warp_reduce16_slot(lane);
                if (!(lane & 1) && slot < 11) atomicAdd(&s_sacc[(s - cs) * kSegAcc + slot], tot);
                if (lane == 0 && nval) atomicAdd(&s_scnt[s - cs], nval);
              };
              begin_segment();
              for (int c = 0; c < nch; ++c) {
                const int st = c % kRingStages;
                mbar_wait(ring_bar + st * 8, (ring_phase >> st) & 1u);
                ring_phase ^= 1u << st;
                const int q0 = r_w0 + c * kGgsUnroll;
                if (q0 + kGgsUnroll <= r_w1 && q0 + kGgsUnroll <= seg_end && (q0 + kGgsUnroll - sd.x) * 32 <= sd.y) {
                  // common case: the whole chunk lies inside the current pair segment and holds no padding rows ->
                  // a branch-free body the compiler interleaves across the four matches
                  float4 pt[kGgsUnroll];
#pragma unroll
                  for (int u = 0; u < kGgsUnroll; ++u) pt[u] = ring_ptr[(st * kGgsUnroll + u) * 32 + lane];
                  if constexpr (kPaired) {  // (pt[u], pt[u+1]) = (X, Y) of one unit: two matches per lane
                    if (kEval) {
#pragma unroll
                      for (int u = 0; u < kGgsUnroll; u += 2) {
                        sampson_match<kEval>(unit_match_a(pt[u], pt[u + 1]), Fm, true, P.smax, g);
                        sampson_match<kEval>(unit_match_b(pt[u], pt[u + 1]), Fm, true, P.smax, g);
                      }
                    } else {
#pragma unroll
                      for (int u = 0; u < kGgsUnroll; u += 2) sampson_match2_unit(pt[u], pt[u + 1], Fm, P.smax, g2);
                    }
                  } else if (kEval) {
#pragma unroll
                    for (int u = 0; u < kGgsUnroll; ++u) sampson_match<kEval>(pt[u], Fm, true, P.smax, g);
                  } else {
#pragma unroll
                    for (int u = 0; u < kGgsUnroll; u += 2) sampson_match2(pt[u], pt[u + 1], Fm, P.smax, g2);
                  }
                } else if constexpr (kPaired) {
#pragma unroll
                  for (int u = 0; u < kGgsUnroll; u += 2) {
                    const int q = q0 + u;  // even; r_w1 and every segment start are even, so the unit is whole
                    if (q < r_w1) {        // warp-uniform
                      if (q >= seg_end) {  // next pair segment (warp-uniform, rare)
                        end_segment();
                        ++s;
                        sd = s_seg[s - cs];
                        seg_end = s_seg[s - cs + 1].x;
                        begin_segment();
                      }
                      const float4 X = ring_ptr[(st * kGgsUnroll + u) * 32 + lane];
                      const float4 Y = ring_ptr[(st * kGgsUnroll + u + 1) * 32 + lane];
                      const bool inb_a = (q - sd.x) * 32 + lane < sd.y, inb_b = (q + 1 - sd.x) * 32 + lane < sd.y;
                      if (kEval) {
                        sampson_match<kEval>(unit_match_a(X, Y), Fm, inb_a, P.smax, g);
                        sampson_match<kEval>(unit_match_b(X, Y), Fm, inb_b, P.smax, g);
                      } else {
                        sampson_match<false, 2>(unit_match_a(X, Y), Fm, inb_a, P.smax, reinterpret_cast<float*>(g2));
                        sampson_match<false, 2>(unit_match_b(X, Y), Fm, inb_b, P.smax, reinterpret_cast<float*>(g2));
                      }
                    }
                  }
                } else {
#pragma unroll
                  for (int u = 0; u < kGgsUnroll; ++u) {
                    const int q = q0 + u;
                    if (q < r_w1) {        // warp-uniform
                      if (q >= seg_end) {  // next pair segment (warp-uniform, rare)
                        end_segment();
                        ++s;
                        sd = s_seg[s - cs];
                        seg_end = s_seg[s - cs + 1].x;
                        begin_segment();
                      }
                      const float4 pt = ring_ptr[(st * kGgsUnroll + u) * 32 + lane];
                      const bool inb = (q - sd.x) * 32 + lane < sd.y;
                      if (kEval) sampson_match<kEval>(pt, Fm, inb, P.smax, g);
                      else sampson_match<false, 2>(pt, Fm, inb, P.smax, reinterpret_cast<float*>(g2));
                    }
                  }
                }
                __syncwarp();  // every lane has consumed the stage before it is refilled
                if (lane == 0 && c + kRingStages < nch) issue(c + kRingStages);
              }
              end_segment();
            }
          } else {
          int s = max(cs, wseg0);
          int r = (s < ce) ? max(r_w0, s_seg[s - cs].x) : r_w1;
          while (s < ce && r < r_w1) {
            const int4 sd = s_seg[s - cs];
            const int r_end = min(r_w1, s_seg[s - cs + 1].x);
            // F' of this pair: 9 lanes x 6 FMAs from the K-folded frame terms, then broadcast
            float Fm[9];
            {
              float mine = 0.f;
              if (lane < 9 && sd.z != sd.w)  // diagonal pair: F' = 0 exactly (reference quirk, see geom.cuh)
                mine = pair_F_entry(s_At + sd.z * 9, s_Rt + sd.z * 9, s_At + sd.w * 9, s_Rt + sd.w * 9, lane / 3, lane % 3);
#pragma unroll
              for (int k = 0; k < 9; ++k) Fm[k] = __shfl_sync(0xffffffffu, mine, k);
              if (kEval && pr.dbg_F && lane < 9) pr.dbg_F[(size_t)s * 9 + lane] = mine;
            }
            float g[16];
#pragma unroll
            for (int k = 0; k < 16; ++k) g[k] = 0.f;
            int nval = 0;
            const int seg_first = sd.x, seg_count = sd.y;
            if (resident) {
              const float4* base = s_pts + (size_t)(r - r_cta0) * 32 + lane;
              const int nr = r_end - r;
              // rounds without padding rows (all but possibly the segment's last one) run a select-free body
              const int n_full = max(0, min(nr, seg_first + seg_count / 32 - r));
              if constexpr (kPaired) {
                // r, r_end and nr are even: the slice is a run of whole units (X = base[q*32], Y = base[(q+1)*32], q even)
                const int n_full2 = n_full & ~1;  // rounds of the leading units without padding rows
                if (kEval) {
                  for (int q = 0; q < nr; q += 2) {
                    const float4 X = base[q * 32], Y = base[(q + 1) * 32];
                    const bool inb_a = (r + q - seg_first) * 32 + lane < seg_count;
                    const bool inb_b = (r + q + 1 - seg_first) * 32 + lane < seg_count;
                    sampson_match<kEval>(unit_match_a(X, Y), Fm, inb_a, P.smax, g);
                    sampson_match<kEval>(unit_match_b(X, Y), Fm, inb_b, P.smax, g);
                  }
                } else {
                  float2 g2[12];
#pragma unroll
                  for (int k = 0; k < 12; ++k) g2[k] = make_float2(0.f, 0.f);
#pragma unroll 2
                  for (int q = 0; q < n_full2; q += 2) sampson_match2_unit(base[q * 32], base[(q + 1) * 32], Fm, P.smax, g2);
                  for (int q = n_full2; q < nr; q += 2) {
                    const float4 X = base[q * 32], Y = base[(q + 1) * 32];
                    const bool inb_a = (r + q - seg_first) * 32 + lane < seg_count;
                    const bool inb_b = (r + q + 1 - seg_first) * 32 + lane < seg_count;
                    sampson_match<false, 2>(unit_match_a(X, Y), Fm, inb_a, P.smax, reinterpret_cast<float*>(g2));
                    sampson_match<false, 2>(unit_match_b(X, Y), Fm, inb_b, P.smax, reinterpret_cast<float*>(g2));
                  }
#pragma unroll
                  for (int k = 0; k < 12; ++k) g[k] = g2[k].x + g2[k].y;
                }
              } else if (kEval) {
#pragma unroll 4
                for (int q = 0; q < n_full; ++q) sampson_match<kEval>(base[q * 32], Fm, true, P.smax, g);
                for (int q = n_full; q < nr; ++q) {
                  const bool inb = (r + q - seg_first) * 32 + lane < seg_count;
                  sampson_match<kEval>(base[q * 32], Fm, inb, P.smax, g);
                }
              } else {  // packed fp32x2 body, two rounds per step; the accumulators live in g2 (x: row A / scalar tail, y: row B)
                float2 g2[12];
#pragma unroll
                for (int k = 0; k < 12; ++k) g2[k] = make_float2(0.f, 0.f);
                int qd = 0;
#pragma unroll 2
                for (; qd + 1 < n_full; qd += 2) sampson_match2(base[qd * 32], base[(qd + 1) * 32], Fm, P.smax, g2);
                for (int q = qd; q < nr; ++q) {
                  const bool inb = (r + q - seg_first) * 32 + lane < seg_count;
                  sampson_match<false, 2>(base[q * 32], Fm, inb, P.smax, reinterpret_cast<float*>(g2));
                }
#pragma unroll
                for (int k = 0; k < 12; ++k) g[k] = g2[k].x + g2[k].y;
              }
            } else {
              // software-pipelined stream: the next batch of kGgsUnroll rounds (2 KB per warp) is requested before the
              // current one is consumed, so up to 2*kGgsUnroll rounds per warp are in flight (HBM latency x bandwidth)
              float4 cur[kGgsUnroll], nxt[kGgsUnroll];
#pragma unroll
              for (int u = 0; u < kGgsUnroll; ++u)
                if (r + u < r_end) cur[u] = ld_stream_f4(pr.pts + (size_t)(r + u) * 32 + lane);
              for (; r < r_end; r += kGgsUnroll) {
#pragma unroll
                for (int u = 0; u < kGgsUnroll; ++u)
                  if (r + kGgsUnroll + u < r_end) nxt[u] = ld_stream_f4(pr.pts + (size_t)(r + kGgsUnroll + u) * 32 + lane);
                if constexpr (kPaired) {  // r and r_end are even: (cur[u], cur[u+1]) = (X, Y) of one whole unit
#pragma unroll
                  for (int u = 0; u < kGgsUnroll; u += 2) {
                    if (r + u < r_end) {  // warp-uniform
                      const bool inb_a = (r + u - seg_first) * 32 + lane < seg_count;
                      const bool inb_b = (r + u + 1 - seg_first) * 32 + lane < seg_count;
                      sampson_match<kEval>(unit_match_a(cur[u], cur[u + 1]), Fm, inb_a, P.smax, g);
                      sampson_match<kEval>(unit_match_b(cur[u], cur[u + 1]), Fm, inb_b, P.smax, g);
                    }
                  }
                } else {
#pragma unroll
                for (int u = 0; u < kGgsUnroll; ++u) {
                  if (r + u < r_end) {  // warp-uniform
                    const bool inb = (r + u - seg_first) * 32 + lane < seg_count;
                    sampson_match<kEval>(cur[u], Fm, inb, P.smax, g);
                  }
                }
                }
#pragma unroll
                for (int u = 0; u < kGgsUnroll; ++u) cur[u] = nxt[u];
              }
            }
            // warp reduction: 16 shuffles for the float slots, one redux for the count
            nval = __reduce_add_sync(0xffffffffu, (int)g[11]);  // per-lane counts are exact small integers
            const float tot = warp_reduce16(g, lane);
            const int slot = warp_reduce16_slot(lane);
            if (!(lane & 1) && slot < 11) atomicAdd(&s_sacc[(s - cs) * kSegAcc + slot], tot);
            if (lane == 0 && nval) atomicAdd(&s_scnt[s - cs], nval);
            r = r_end;
            ++s;
          }
          }
        }
        __syncthreads();
        if (kProbe && pr.dbg_clock && tid == 0) ck1a = clock64();
        // ---- stage 2a: per-pair adjoint, one warp per segment, 18 lanes x 2 outputs; leaves the slots zeroed ----
        for (int sl = warp; sl < nchunk; sl += kGgsWarps) {
          const int4 sd = s_seg[sl];
          float* G = s_sacc + sl * kSegAcc;
          float g3[3] = {0.f, 0.f, 0.f}, gs = 0.f;
          const int side = lane >= 9, e = (lane - side * 9) % 9, i = e / 3, j = e - i * 3;
          if (lane < 18) {
#pragma unroll
            for (int k = 0; k < 3; ++k) g3[k] = side ? G[k * 3 + i] : G[i * 3 + k];
            if (kEval && pr.dbg_G && lane < 9) atomicAdd(&pr.dbg_G[(size_t)(cs + sl) * 9 + lane], G[lane]);
          } else if (lane < 20) {
            gs = G[9 + (lane - 18)];
          }
          const int cnt_seg = s_scnt[sl];
          __syncwarp();
          if (lane < kSegAcc) G[lane] = 0.f;
          if (lane == 0) s_scnt[sl] = 0;
          if (lane < 18) {
            const int self = side ? sd.w : sd.z, other = side ? sd.z : sd.w;
            float oA, oR;
            pair_adjoint_entry(g3, s_At + other * 9, s_Rt + other * 9, j, &oA, &oR);
            atomicAdd(&s_fg[self * 18 + e], oA);
            atomicAdd(&s_fg[self * 18 + 9 + e], oR);
          } else if (lane == 18) {
            atomicAdd(&s_misc[4], gs);
            atomicAdd(&s_cta_cnt, cnt_seg);
          } else if (lane == 19 && kEval) {
            atomicAdd(&s_misc[5], gs);
          }
        }
      }
      __syncthreads();
      if (kProbe && pr.dbg_clock && tid == 0) ck1 = clock64();
      // ================= stage 2b: one thread per frame: unfold K, frame adjoint -> the CTA's partial gradient =================
      if (warp * 32 < N) {  // the warps that hold frames (one thread per frame)
        const int n = tid;
        float k4[4] = {0.f, 0.f, 0.f, 0.f};
        if (n < N) {
          float* gAt = s_fg + n * 18;
          float gT[3] = {0.f, 0.f, 0.f}, gq[4] = {0.f, 0.f, 0.f, 0.f};
          if (s_mine[n]) {  // the frames this CTA's segments touch (static plan); all other slots stay zero
            float gA[9], gR[9];
            frame_unfold(s_A + n * 9, s_R + n * 9, kin, gAt, gAt + 9, gA, gR, k4);
            frame_adjoint(s_pose + n * 9, s_R + n * 9, gR, gA, gT, gq);
#pragma unroll
            for (int k = 0; k < 18; ++k) gAt[k] = 0.f;
          }
#pragma unroll
          for (int k = 0; k < 3; ++k) s_part[n * 7 + k] = gT[k];
#pragma unroll
          for (int k = 0; k < 4; ++k) s_part[n * 7 + 3 + k] = gq[k];
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) k4[k] = warp_sum(k4[k]);  // d/d(ix, iy, kx, ky) summed over the warp's frames
        if (lane == 0) {
          if (N <= 32) {
#pragma unroll
            for (int k = 0; k < 4; ++k) s_misc[8 + k] = k4[k];
          } else {
#pragma unroll
            for (int k = 0; k < 4; ++k) atomicAdd(&s_misc[8 + k], k4[k]);
          }
        }
      }
      __syncthreads();
      if (kProbe && pr.dbg_clock && tid == 0) ck2 = clock64();
      // ================= exchange: all-reduce of the partial gradient over the CTAs of this sequence =================
      ggs_exchange<kEval>(pr.xch1, pr.xch2, P.xch_mode == 1 ? pr.acc : nullptr, cpp, cta, P.xch_group, N, it_global, s_part, s_misc, s_cta_cnt,
                          (-s_misc[8] + cx * s_misc[10]) / (fpx * fpx), (-s_misc[9] + cy * s_misc[11]) / (fpy * fpy), s_gsum, s_expect, s_mine);
      ++it_global;
      __syncthreads();
      if (kProbe && pr.dbg_clock && tid == 0) {
        ck3 = clock64();
        clk_sum[1] += ck1a - ck0; clk_sum[4] += ck1 - ck1a; clk_sum[2] += ck2 - ck1; clk_sum[3] += ck3 - ck2; clk_sum[5] += 1;
      }
      // ================= stage 3: finish the step, all threads (identical in every CTA) =================
      bool drop_phase = false;
      {
        const int n_valid = __float_as_int(s_gsum[N * 7 + 4]);
        last_valid = n_valid;
        last_logged = s_gsum[N * 7 + 2] * inv_m_total;
        // len(valid) / N < min_matches  (:103-105), evaluated as n < min_matches * N in float64
        drop_phase = !kEval && (P.min_matches > 0.0) && ((double)n_valid < P.min_matches * (double)N);
        if (tid == 0) {  // the CTA-level partial sums are consumed: zero them for the next iteration (written after >= 1 barrier)
          s_misc[4] = 0.f; s_misc[5] = 0.f;
          s_misc[8] = 0.f; s_misc[9] = 0.f; s_misc[10] = 0.f; s_misc[11] = 0.f;
          s_cta_cnt = 0;
        }
        if (drop_phase) {
          dropped = 1;
        } else {
          const float inv_n = 1.0f / (float)n_valid;  // mean over the valid matches (:110)
          const float gfx = upd_FL ? s_gsum[N * 7 + 0] * scale_over_N : 0.f;
          const float gfy = upd_FL ? s_gsum[N * 7 + 1] * scale_over_N : 0.f;
          auto grad_of = [&](int e) {  // d mean(valid err) / d pose[e]
            const int n = e / 9, c = e - n * 9;
            float gsum;
            if (c < 3) gsum = upd_T ? s_gsum[n * 7 + c] : 0.f;
            else if (c < 7) gsum = upd_R ? s_gsum[n * 7 + c] : 0.f;
            else gsum = (c == 7 ? gfx : gfy) * s_fl[n * 2 + (c - 7)] * s_inr[n * 2 + (c - 7)];
            return gsum * inv_n;
          };
          if (kEval) {
            if (cta == 0) {
              for (int e = tid; e < N9; e += kGgsThreads) pr.dbg_grad[e] = grad_of(e);
              if (tid == 0) {
                pr.dbg_scalars[0] = s_gsum[N * 7 + 3] / (float)n_valid;
                pr.dbg_scalars[1] = (float)n_valid;
                pr.dbg_scalars[2] = last_logged;
                pr.dbg_scalars[3] = 0.f;
              }
            }
          } else {
            // clip norms: one element per thread (N9 <= 1152: up to three), warp sums, partials through shared memory
            constexpr int kPer = (kMaxFrames * 9 + kGgsThreads - 1) / kGgsThreads;
            float gv[kPer];
            float gn2 = 0.f, pn2 = 0.f;
#pragma unroll
            for (int q = 0; q < kPer; ++q) {
              const int e = tid + q * kGgsThreads;
              gv[q] = 0.f;
              if (e < N9) {
                const float g1 = grad_of(e);
                gv[q] = g1;
                gn2 = fmaf(g1, g1, gn2);
                const float pm = (fabsf(g1) > 0.f) ? s_pose[e] : 0.f;  // grad_mask = grads.abs() > 0 (:117)
                pn2 = fmaf(pm, pm, pn2);
              }
            }
            const int warps_used = min(kGgsWarps, (N9 + 31) / 32);  // warps that hold elements (the others contribute zeros)
            if (warp < warps_used) {
              gn2 = warp_sum(gn2);
              pn2 = warp_sum(pn2);
              if (lane == 0) {
                s_misc[16 + warp * 2] = gn2;
                s_misc[16 + warp * 2 + 1] = pn2;
              }
            }
            __syncthreads();
            if (kProbe && pr.dbg_clock && tid == 0) { const long long c = clock64(); clk_sum[0] += c - ck3; ck3 = c; }  // probe: norm partials
            gn2 = 0.f;
            pn2 = 0.f;
            for (int wv = 0; wv < warps_used; ++wv) {  // fixed order: identical in every thread and CTA
              gn2 += s_misc[16 + wv * 2];
              pn2 += s_misc[16 + wv * 2 + 1];
            }
            const float max_norm = alpha_over_lr * sqrtf(pn2);       // alpha * |x . mask| / lr  (:119)
            const float cc = max_norm / (sqrtf(gn2) + 1e-6f);        // clip_grad_norm_
            const float coef = (cc > 1.0f) ? 1.0f : cc;              // clamp(max=1), NaN passes through
#pragma unroll
            for (int q = 0; q < kPer; ++q) {
              const int e = tid + q * kGgsThreads;
              if (e < N9) {
                const float g1 = gv[q] * coef;
                const float v = (done == 0) ? g1 : fmaf(P.momentum, s_vel[e], g1);  // momentum buffer resets per phase
                s_vel[e] = v;
                const float pnew = s_pose[e] - P.lr * v;
                s_pose[e] = pnew;
                const int n = e / 9, c = e - n * 9;
                if (c >= 7) focal_of(pnew, &s_fl[n * 2 + (c - 7)], &s_inr[n * 2 + (c - 7)]);
              }
            }
            ++done;
            __syncthreads();
            if (kProbe && pr.dbg_clock && tid == 0) { const long long c = clock64(); clk_sum[7] += c - ck3; ck3 = c; }  // probe: coefficient + update
            frames_forward();  // stage 0 of the next iteration (one block barrier inside)
          }
        }
      }
      if (kProbe && pr.dbg_clock && tid == 0) clk_sum[6] += clock64() - ck3;
      if (kEval) break;
      if (drop_phase) break;  // uniform: phase dropped on "insufficient valid matches" (no update, :103-108)
    }
    if (kEval) break;
    if (tid == 0 && cta == 0 && pr.stats) {
      pr.stats->sampson[phase] = last_logged;
      pr.stats->iters[phase] = done;
      pr.stats->dropped[phase] = dropped;
      pr.stats->n_valid[phase] = last_valid;
    }
  }
  if (kProbe && pr.dbg_clock && tid == 0)
    for (int k = 0; k < 8; ++k) pr.dbg_clock[(size_t)cta * 8 + k] += clk_sum[k];
  if (!kEval && cta == 0) {
    for (int e = tid; e < N9; e += kGgsThreads) pr.pose[e] = s_pose[e];
  }
}

}  // namespace pdb
