// Denoiser forward + DDPM posterior update as ONE persistent cooperative kernel per launch
// (models/denoiser.py:53-76, util/embedding.py:13-50, models/gaussian_diffuser.py:190-282).
//
// A launch runs diffusion steps t_hi .. t_lo back to back.  Per step the grid walks 43 stages separated by
// group barriers: embed+first, 8 x (LN1+QKV, attention, out-proj+residual, LN2+FF1+ReLU, FF2+residual),
// last0, tail (LayerNorm(128)+ReLU+Linear(128->9) fused with x0 / posterior mean / noise add).
// Loop-invariant work is hoisted: z-projection (385 of the 702 `_first` input columns) once per launch,
// the timestep-embedding MLP and its `_first` block once per weight load (table of 100 rows).
//
// This file is the exact-fp32 engine: CUDA-core FMAs, weights re-laid out k4-major ([K/4][O] float4) so that a
// warp reads 512 contiguous bytes per step while every lane owns one output feature; activations of a token tile
// are staged in shared memory and broadcast.  S = B*N tokens is tiny (20..160 per GPU): every stage is
// latency / weight-bandwidth bound (SURVEY.md §8d).
//
// Stage hand-over, two instantiations of the same kernel (kFlag = false is the product default; kFlag = true is bit-identical
// in its results and slower -- every CTA polls the 80 KB flagged tile through L2, see tools/stage_probe.cu -- and stays as a tested alternative behind pdb_debug_denoiser_handover):
//   kFlag = false  activations are plain floats in global memory; a group barrier (block barrier, release reduction,
//                  acquire poll) separates consecutive stages.
//   kFlag = true   every activation is published as ONE 64-bit word {fp32 value, 32-bit version tag} with a relaxed store
//                  (single-copy atomic: a reader that sees the tag has the value that was stored with it).  A consumer loads
//                  the words of the tile it needs and re-loads those whose tag is not the expected version yet: there is NO
//                  barrier, no fence and no counter between stages -- the data is its own flag (the protocol NCCL calls LL).
//                  Write-after-read safety needs no synchronisation either: every reader of a buffer version is, through the
//                  data it produces, a dependency of the item that overwrites it (argument per buffer in DESIGN.md §4.2); the
//                  one buffer for which this fails, qkv (an attention item reads key rows of OTHER token tiles), is double
//                  buffered by layer parity.
#pragma once
#include <type_traits>

#include "common.cuh"
#include "posediff_b200.h"

namespace pdb {

constexpr int kDM = 512;       // d_model            (cfgs/default.yaml:28)
constexpr int kHeads = 4;      // nhead              (:29)
constexpr int kHD = 128;       // head dim
constexpr int kFF = 1024;      // dim_feedforward    (:30)
constexpr int kLayers = 8;     // num_encoder_layers (:31)
constexpr int kHid = 128;      // mlp_hidden_dim     (denoiser.py:29)
constexpr int kZ = 384;
constexpr int kTEmb = 128;
constexpr int kPoseEmb = 189;  // 9 * (2*10 + 1)
constexpr int kPoseEmbPad = 256;  // 189 harmonic-pose columns zero-padded so that K/4 splits over 32 k-slices
constexpr int kFirstIn = 702;
constexpr int kT = PDB_NUM_TIMESTEPS;
constexpr int kDenThreads = 256;
constexpr int kDenWarps = kDenThreads / 32;
constexpr float kLnEps = 1e-5f;

struct LayerWeights {
  const float4* w_qkv;  // packed [512/4][1536]
  const float* b_qkv;
  const float4* w_out;  // [512/4][512]
  const float* b_out;
  const float4* w_ff1;  // [512/4][1024]
  const float* b_ff1;
  const float4* w_ff2;  // [1024/4][512]
  const float* b_ff2;
  const float *ln1_g, *ln1_b, *ln2_g, *ln2_b;
};

struct DenoiserDev {  // device pointers into the packed weight arena
  const float4* w_first_x;  // [256/4][512]  (harmonic-pose columns 0..188 of _first.weight, zero padded)
  const float4* w_first_z;  // [384/4][512]  (columns 317..700)
  const float* w_first_pivot;  // [512]      (column 701)
  const float* b_first;        // [512]
  const float* tproj;          // [100][512]  = t_emb(t) @ _first.weight[:,189:317]^T
  LayerWeights layer[kLayers];
  const float4* w_last0;  // [512/4][128]
  const float* b_last0;
  const float *ln_last_g, *ln_last_b;
  const float* w_last3;  // [9][128] row-major (as in the checkpoint)
  const float* b_last3;
  const float* sched;    // [100][8]: a_t, b_t, c1_t, c2_t, sigma_t
};

struct DenoiserRun {
  int batch, frames, tokens;
  int t_hi, t_lo;          // steps t_hi, t_hi-1, ..., t_lo
  int guide_below;         // t < guide_below: leave the posterior mean in x (no noise; the GGS kernel follows)
  int compute_zproj;       // 1: (re)compute the z projection at the start of this launch
  float* x;                // [S,9] sampler state, updated in place
  const float* z;          // [S,384]
  const float* draws;      // [T+1,S,9] or null (no noise added)
  float* trail;            // [T+1,S,9] or null
  float* eps_out;          // [S,9] or null (network output of the LAST step run)
  float* x0_out;           // [S,9] or null
  float* mean_out;         // [S,9] or null
  // workspace
  float *zproj, *h, *qkv, *att, *ff, *u;
  unsigned* bar;           // zero on entry
  // kFlag kernels: flag-carrying activation buffers (64-bit {fp32, tag} words) and the first tag of this launch.
  // fqkv holds two buffers [2][S][1536] (layer parity); fx [S][16] shadows x between the steps of one launch.
  unsigned long long *fh, *fqkv, *fatt, *fff, *fu, *fx;
  unsigned tag_base;       // versions of this launch are tag_base + step * kTagsPerStep + id; all larger than any earlier launch's
  long long* dbg_clock;    // may be null: [ctas][8] cycle sums {barrier, tile load + LayerNorm, linear item, attention, tail, steps}
};

inline size_t denoiser_ws_floats(int tokens) {
  return (size_t)tokens * (kDM + kDM + 3 * kDM + kDM + kFF + kHid) + 64;
}
// 64-bit words of the flag-carrying buffers (fh, fqkv x 2, fatt, fff, fu, fx)
constexpr int kTagsPerStep = 64;  // version ids of one diffusion step: 0 first, 1+5l qkv, 2+5l att, 3+5l out-proj, 4+5l ff, 5+5l FF2, 41 u, 42 x
inline size_t denoiser_flag_ws_words(int tokens) {
  return (size_t)tokens * (kDM + 2 * 3 * kDM + kDM + kFF + kHid + 16);
}

// ---------------------------------------------------------------------------------------------
// token-tile loaders (global -> shared), one warp per row
// ---------------------------------------------------------------------------------------------
// LayerNorm of the staged rows (shared memory, one warp per row)
template <int K, int TS>
__device__ __forceinline__ void layer_norm_rows(float* __restrict__ Xs, int row0, int valid_end, const float* __restrict__ ln_g,
                                                const float* __restrict__ ln_b) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int PL = K / 128;  // float4 per lane per row
  for (int r = warp; r < TS; r += kDenWarps) {
    if (row0 + r >= valid_end) continue;
    float4* row = reinterpret_cast<float4*>(Xs + (size_t)r * K);
    float4 x[PL];
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < PL; ++i) {
      x[i] = row[lane + 32 * i];
      sum += x[i].x + x[i].y + x[i].z + x[i].w;
    }
    const float mean = warp_sum(sum) * (1.0f / K);
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < PL; ++i) {
      x[i].x -= mean; x[i].y -= mean; x[i].z -= mean; x[i].w -= mean;
      sq += x[i].x * x[i].x + x[i].y * x[i].y + x[i].z * x[i].z + x[i].w * x[i].w;
    }
    const float rstd = 1.0f / sqrtf(warp_sum(sq) * (1.0f / K) + kLnEps);
#pragma unroll
    for (int i = 0; i < PL; ++i) {
      const float4 g = __ldg(reinterpret_cast<const float4*>(ln_g) + lane + 32 * i);
      const float4 b = __ldg(reinterpret_cast<const float4*>(ln_b) + lane + 32 * i);
      x[i].x = x[i].x * rstd * g.x + b.x;
      x[i].y = x[i].y * rstd * g.y + b.y;
      x[i].z = x[i].z * rstd * g.z + b.z;
      x[i].w = x[i].w * rstd * g.w + b.w;
      row[lane + 32 * i] = x[i];
    }
  }
}

// plain copy or LayerNorm of a [rows, K] slab; rows >= valid are zero-filled.  All global loads of the tile are
// issued before any is consumed (ONE L2 round trip per stage); the LayerNorm then runs out of shared memory.
template <int K, int TS>
__device__ __forceinline__ void load_rows(float* __restrict__ Xs, const float* __restrict__ src, int row0, int valid_end,
                                          const float* __restrict__ ln_g, const float* __restrict__ ln_b) {
  constexpr int K4 = K / 4;
  constexpr int TOTAL = TS * K4;                    // float4 elements of the tile
  constexpr int PER = (TOTAL + kDenThreads - 1) / kDenThreads;
  float4 v[PER];
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    const int idx = threadIdx.x + i * kDenThreads;
    const int r = idx / K4, c = idx - r * K4;
    v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (idx < TOTAL && row0 + r < valid_end) v[i] = __ldcg(reinterpret_cast<const float4*>(src + (size_t)(row0 + r) * K) + c);
  }
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    const int idx = threadIdx.x + i * kDenThreads;
    if (idx < TOTAL) reinterpret_cast<float4*>(Xs)[idx] = v[i];
  }
  if (ln_g) {
    __syncthreads();
    layer_norm_rows<K, TS>(Xs, row0, valid_end, ln_g, ln_b);
  }
}

// The same tile out of flag-carrying words: [rows, K] words of version `tag`.  All loads of a batch are in flight together
// (one L2 round trip when the producers are done); a word whose tag is not there yet is simply loaded again.
__device__ __forceinline__ bool ll_ready(unsigned long long w, unsigned tag) { return (unsigned)(w >> 32) == tag; }
__device__ __forceinline__ float ll_value(unsigned long long w) { return __uint_as_float((unsigned)w); }

template <int K, int TS>
__device__ __forceinline__ void load_rows_flag(float* __restrict__ Xs, const unsigned long long* __restrict__ src, int row0,
                                               int valid_end, unsigned tag, const float* __restrict__ ln_g,
                                               const float* __restrict__ ln_b) {
  constexpr int K2 = K / 2;                                    // 16-byte word pairs per row
  constexpr int TOTAL = TS * K2;
  constexpr int PER = (TOTAL + kDenThreads - 1) / kDenThreads;
  constexpr int ROUNDS = (PER + 19) / 20;                      // at most 20 pairs (80 registers) in flight per thread
  constexpr int BATCH = (PER + ROUNDS - 1) / ROUNDS;
#pragma unroll 1
  for (int round = 0; round < ROUNDS; ++round) {
    unsigned long long a[BATCH], b[BATCH];
#pragma unroll
    for (int i = 0; i < BATCH; ++i) {
      const int idx = threadIdx.x + (round * BATCH + i) * kDenThreads;
      const int r = idx / K2, c = idx - r * K2;
      a[i] = b[i] = (unsigned long long)tag << 32;             // rows beyond the valid range: zeros, "ready"
      if (idx < TOTAL && row0 + r < valid_end) ld_ll2(src + (size_t)(row0 + r) * K + 2 * c, a[i], b[i]);
    }
#pragma unroll
    for (int i = 0; i < BATCH; ++i) {
      const int idx = threadIdx.x + (round * BATCH + i) * kDenThreads;
      const int r = idx / K2, c = idx - r * K2;
      if (idx < TOTAL) {
        while (!ll_ready(a[i], tag) || !ll_ready(b[i], tag)) {
          ll_backoff();
          ld_ll2(src + (size_t)(row0 + r) * K + 2 * c, a[i], b[i]);
        }
        reinterpret_cast<float2*>(Xs)[idx] = make_float2(ll_value(a[i]), ll_value(b[i]));
      }
    }
  }
  if (ln_g) {
    __syncthreads();
    layer_norm_rows<K, TS>(Xs, row0, valid_end, ln_g, ln_b);
  }
}

// harmonic pose embedding (pytorch3d HarmonicEmbedding, n=10, logspace, append_input; embedding.py:44):
// [sin(x_c 2^k) (c-major) | cos(same) | x | 0 0 0]
// The tile's x rows are staged in `xrow` first: plain x at the first step of a launch (written by the previous kernel), the
// flag-carrying shadow fx (version `tag`, written by the previous step's tail) afterwards in the kFlag kernels.
__device__ __forceinline__ void load_pose_embed(float* __restrict__ Xs, float* __restrict__ xrow, const float* __restrict__ x,
                                                const unsigned long long* __restrict__ fx, unsigned tag, int row0, int rows,
                                                int valid_end) {
  for (int i = threadIdx.x; i < rows * kTargetDim; i += kDenThreads) {
    const int r = i / kTargetDim, c = i - r * kTargetDim;
    const int s = row0 + r;
    float v = 0.f;
    if (s < valid_end) {
      if (fx) {
        unsigned long long w = ld_ll(fx + (size_t)s * 16 + c);
        while (!ll_ready(w, tag)) {
          ll_backoff();
          w = ld_ll(fx + (size_t)s * 16 + c);
        }
        v = ll_value(w);
      } else {
        v = __ldcg(x + (size_t)s * kTargetDim + c);
      }
    }
    xrow[i] = v;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < rows * kPoseEmbPad; i += kDenThreads) {
    const int r = i / kPoseEmbPad, col = i - r * kPoseEmbPad;
    const int s = row0 + r;
    float v = 0.f;
    if (s < valid_end && col < kPoseEmb) {
      if (col < 180) {
        const int j = col < 90 ? col : col - 90;
        const int c = j / 10, k = j - c * 10;
        const float arg = xrow[r * kTargetDim + c] * (float)(1 << k);
        v = col < 90 ? sinf(arg) : cosf(arg);
      } else {
        v = xrow[r * kTargetDim + (col - 180)];
      }
    }
    Xs[i] = v;
  }
}

// ---------------------------------------------------------------------------------------------
// One linear work item: 32 output features x one token tile.  Xs = staged activations [TS][K].
// ---------------------------------------------------------------------------------------------
enum : int { kEpiNone = 0, kEpiRelu = 1, kEpiSilu = 2 };

// Work item of a linear stage: kFPI = 8 output features x one token tile, so that even the narrow stages
// (512 outputs -> 64 items) spread over many SMs.  Inside the CTA the reduction dimension is cut into 32 k-slices:
// lane = (ks = lane>>3, f = lane&7), slice = warp*4 + ks owns the k4-rows  i*32 + slice.  A warp-load of weights
// touches 4 k4-rows x 128 contiguous bytes; the 4 k-slices of a warp read 64 contiguous bytes of the staged
// activations (broadcast to the 8 feature lanes).
constexpr int kFPI = 8;
constexpr int kSlices = kDenWarps * 4;

template <int K>
struct LinW {
  static constexpr int K4 = K / 4;
  static constexpr int PER = K4 / kSlices;
  static_assert(K4 % kSlices == 0 && PER >= 1 && PER <= 16, "K layout");
  float4 w[PER];
};

// Issue the weight loads of one work item.  Weights never depend on activations, so this is called BEFORE the group
// barrier that precedes the stage: the L2 latency of the weight stream hides behind the barrier.
template <int K>
__device__ __forceinline__ void linear_prefetch(LinW<K>& W, const float4* __restrict__ Wp, int O, int o0) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int slice = warp * 4 + (lane >> 3);
  const float4* wp = Wp + (size_t)slice * O + o0 + (lane & 7);
#pragma unroll
  for (int i = 0; i < LinW<K>::PER; ++i) W.w[i] = __ldg(wp + (size_t)i * kSlices * O);
}

// Epilogue of a linear stage: Y = epi(acc + bias + add1[row, o] + add2[o] + add_rs[o] * rs[row]).  add1 / Y are plain float
// arrays, or (kFlag kernels, add1_flag / y_flag) arrays of flag-carrying words; Y is then published with version `tag`.
// A flagged add1 is only ever the value this very thread stored earlier (the residual stream is updated in place by the same
// (item, thread) mapping), so it needs no tag check.
struct LinEpi {
  const float* bias;
  const void* add1;
  int ld1;
  bool add1_flag;
  const float* add2;
  const float* add_rs;
  const float* rs;
  void* Y;
  int ldy;
  bool y_flag;
  int epi;
  unsigned tag;
};

template <int TS, int K, bool kFlag>
__device__ __forceinline__ void linear_item(const LinW<K>& W, const float* __restrict__ Xs, float* __restrict__ red, int o0,
                                            const LinEpi& E, int row0, int valid_end) {
  static_assert(TS % 4 == 0 && TS <= 32, "token tile");
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int PER = LinW<K>::PER;
  const int ks = lane >> 3, f = lane & 7;
  // epilogue operands of this thread's output (token s_out, feature f_out) are requested before the FMA loop
  const int s_out = threadIdx.x >> 3, f_out = threadIdx.x & 7;
  const bool has_out = s_out < TS && (row0 + s_out) < valid_end;
  float epi_add = 0.f;
  if (has_out) {
    const int row = row0 + s_out, o = o0 + f_out;
    if (E.bias) epi_add += __ldg(E.bias + o);
    if (E.add1) {
      if (kFlag && E.add1_flag) epi_add += ll_value(ld_ll(static_cast<const unsigned long long*>(E.add1) + (size_t)row * E.ld1 + o));
      else epi_add += __ldcg(static_cast<const float*>(E.add1) + (size_t)row * E.ld1 + o);
    }
    if (E.add2) epi_add += __ldg(E.add2 + o);
    if (E.add_rs) epi_add += __ldg(E.add_rs + o) * E.rs[s_out];
  }
  float acc[TS];
#pragma unroll
  for (int s = 0; s < TS; ++s) acc[s] = 0.f;
  const float* xs = Xs + (warp * 4 + ks) * 4;
#pragma unroll
  for (int i = 0; i < PER; ++i) {
#pragma unroll
    for (int s = 0; s < TS; ++s) {
      const float4 xv = *reinterpret_cast<const float4*>(xs + s * K + i * kSlices * 4);
      acc[s] = fmaf(W.w[i].x, xv.x, fmaf(W.w[i].y, xv.y, fmaf(W.w[i].z, xv.z, fmaf(W.w[i].w, xv.w, acc[s]))));
    }
  }
  // reduce over the 4 k-slices of the warp: after two exchange steps lane (ks, f) owns tokens ks*TS/4 .. +TS/4-1
  constexpr int Q = TS / 4;
  {
    const bool hi = ks & 2;
#pragma unroll
    for (int s = 0; s < TS / 2; ++s) {
      const float send = hi ? acc[s] : acc[s + TS / 2];
      const float keep = hi ? acc[s + TS / 2] : acc[s];
      acc[s] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
    }
  }
  {
    const bool hi = ks & 1;
#pragma unroll
    for (int s = 0; s < Q; ++s) {
      const float send = hi ? acc[s] : acc[s + Q];
      const float keep = hi ? acc[s + Q] : acc[s];
      acc[s] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
    }
  }
#pragma unroll
  for (int s = 0; s < Q; ++s) red[(warp * TS + ks * Q + s) * kFPI + f] = acc[s];
  __syncthreads();
  if (s_out < TS) {
    float v = 0.f;
#pragma unroll
    for (int wv = 0; wv < kDenWarps; ++wv) v += red[(wv * TS + s_out) * kFPI + f_out];
    if (has_out) {
      v += epi_add;
      if (E.epi == kEpiRelu) v = fmaxf(v, 0.f);
      else if (E.epi == kEpiSilu) v = v / (1.0f + expf(-v));
      const size_t at = (size_t)(row0 + s_out) * E.ldy + o0 + f_out;
      if (kFlag && E.y_flag) st_ll(static_cast<unsigned long long*>(E.Y) + at, __float_as_uint(v), E.tag);
      else static_cast<float*>(E.Y)[at] = v;
    }
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------
// Self-attention for one (sequence, head): N <= 128 keys, head dim 128, fp32.
// ---------------------------------------------------------------------------------------------
// four consecutive flag-carrying words (32-byte aligned) -> float4, polling for version `tag`
__device__ __forceinline__ float4 ld_ll_f4(const unsigned long long* p, unsigned tag) {
  unsigned long long w0, w1, w2, w3;
  ld_ll2(p, w0, w1);
  ld_ll2(p + 2, w2, w3);
  while (!ll_ready(w0, tag) || !ll_ready(w1, tag) || !ll_ready(w2, tag) || !ll_ready(w3, tag)) {
    ll_backoff();
    ld_ll2(p, w0, w1);
    ld_ll2(p + 2, w2, w3);
  }
  return make_float4(ll_value(w0), ll_value(w1), ll_value(w2), ll_value(w3));
}

template <bool kFlag>
__device__ __forceinline__ void attention_item(float* __restrict__ smem, const void* __restrict__ qkv_any, void* __restrict__ att_any,
                                               int seq, int head, int chunk, int N, unsigned tag_in, unsigned tag_out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int KP = kHD + 4;  // padded key rows (float4 aligned): lane = key index reads hit distinct banks
  float* Ks = smem;                        // [N][132]
  float* Vs = Ks + N * KP;                 // [N][128]
  float* Qs = Vs + N * kHD;                // [warps][128]
  float* Ps = Qs + kDenWarps * kHD;        // [warps][128]
  const int i = chunk * kDenWarps + warp;  // this warp's query row
  float4 qv = make_float4(0.f, 0.f, 0.f, 0.f);
  if constexpr (kFlag) {
    const unsigned long long* base = static_cast<const unsigned long long*>(qkv_any) + (size_t)seq * N * (3 * kDM) + head * kHD;
    // keys and values: all loads of up to four elements per thread are issued before the first tag is examined
    const int total = N * (kHD / 4);
    for (int e0 = threadIdx.x; e0 < total; e0 += 4 * kDenThreads) {
      unsigned long long kw[4][4], vw[4][4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int e = e0 + u * kDenThreads;
        if (e < total) {
          const int j = e / (kHD / 4), d4 = e - j * (kHD / 4);
          const unsigned long long* kp = base + (size_t)j * 3 * kDM + kDM + d4 * 4;
          const unsigned long long* vp = base + (size_t)j * 3 * kDM + 2 * kDM + d4 * 4;
          ld_ll2(kp, kw[u][0], kw[u][1]);
          ld_ll2(kp + 2, kw[u][2], kw[u][3]);
          ld_ll2(vp, vw[u][0], vw[u][1]);
          ld_ll2(vp + 2, vw[u][2], vw[u][3]);
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int e = e0 + u * kDenThreads;
        if (e < total) {
          const int j = e / (kHD / 4), d4 = e - j * (kHD / 4);
          const unsigned long long* kp = base + (size_t)j * 3 * kDM + kDM + d4 * 4;
          const unsigned long long* vp = base + (size_t)j * 3 * kDM + 2 * kDM + d4 * 4;
          while (!ll_ready(kw[u][0], tag_in) || !ll_ready(kw[u][1], tag_in) || !ll_ready(kw[u][2], tag_in) || !ll_ready(kw[u][3], tag_in)) {
            ll_backoff();
            ld_ll2(kp, kw[u][0], kw[u][1]);
            ld_ll2(kp + 2, kw[u][2], kw[u][3]);
          }
          while (!ll_ready(vw[u][0], tag_in) || !ll_ready(vw[u][1], tag_in) || !ll_ready(vw[u][2], tag_in) || !ll_ready(vw[u][3], tag_in)) {
            ll_backoff();
            ld_ll2(vp, vw[u][0], vw[u][1]);
            ld_ll2(vp + 2, vw[u][2], vw[u][3]);
          }
          *reinterpret_cast<float4*>(Ks + j * KP + d4 * 4) = make_float4(ll_value(kw[u][0]), ll_value(kw[u][1]), ll_value(kw[u][2]), ll_value(kw[u][3]));
          *reinterpret_cast<float4*>(Vs + j * kHD + d4 * 4) = make_float4(ll_value(vw[u][0]), ll_value(vw[u][1]), ll_value(vw[u][2]), ll_value(vw[u][3]));
        }
      }
    }
    if (i < N) qv = ld_ll_f4(base + (size_t)i * 3 * kDM + lane * 4, tag_in);
  } else {
    const float* base = static_cast<const float*>(qkv_any) + (size_t)seq * N * (3 * kDM) + head * kHD;
    if (i < N) qv = __ldcg(reinterpret_cast<const float4*>(base + (size_t)i * 3 * kDM) + lane);
    for (int e = threadIdx.x; e < N * (kHD / 4); e += kDenThreads) {
      const int j = e / (kHD / 4), d4 = e - j * (kHD / 4);
      const float4 kv = __ldcg(reinterpret_cast<const float4*>(base + (size_t)j * 3 * kDM + kDM) + d4);
      const float4 vv = __ldcg(reinterpret_cast<const float4*>(base + (size_t)j * 3 * kDM + 2 * kDM) + d4);
      *reinterpret_cast<float4*>(Ks + j * KP + d4 * 4) = kv;
      *reinterpret_cast<float4*>(Vs + j * kHD + d4 * 4) = vv;
    }
  }
  const float scaling = 0.08838834764831845f;  // 1/sqrt(128): q is scaled before QK^T (torch MHA)
  *reinterpret_cast<float4*>(Qs + warp * kHD + lane * 4) = make_float4(qv.x * scaling, qv.y * scaling, qv.z * scaling, qv.w * scaling);
  __syncthreads();
  if (i < N) {
    float sc[4];  // up to 128 keys: 4 passes of 32
    float mx = -INFINITY;
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const int j = p * 32 + lane;
      float dot = -INFINITY;
      if (p * 32 < N && j < N) {
        const float4* kr = reinterpret_cast<const float4*>(Ks + j * KP);
        const float4* qr = reinterpret_cast<const float4*>(Qs + warp * kHD);
        float d0 = 0.f, d1 = 0.f, d2 = 0.f, d3 = 0.f;
#pragma unroll 8
        for (int d = 0; d < kHD / 4; ++d) {
          const float4 a = qr[d], b = kr[d];
          d0 = fmaf(a.x, b.x, d0); d1 = fmaf(a.y, b.y, d1); d2 = fmaf(a.z, b.z, d2); d3 = fmaf(a.w, b.w, d3);
        }
        dot = (d0 + d1) + (d2 + d3);
      }
      sc[p] = dot;
      mx = fmaxf(mx, dot);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const int j = p * 32 + lane;
      const float e = (j < N) ? expf(sc[p] - mx) : 0.f;
      sc[p] = e;
      sum += e;
    }
    sum = warp_sum(sum);
    const float inv = 1.0f / sum;
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const int j = p * 32 + lane;
      if (j < N) Ps[warp * kHD + j] = sc[p] * inv;
    }
    __syncwarp();
    float4 o4 = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int j = 0; j < N; ++j) {
      const float pj = Ps[warp * kHD + j];
      const float4 vv = *reinterpret_cast<const float4*>(Vs + j * kHD + lane * 4);
      o4.x = fmaf(pj, vv.x, o4.x); o4.y = fmaf(pj, vv.y, o4.y); o4.z = fmaf(pj, vv.z, o4.z); o4.w = fmaf(pj, vv.w, o4.w);
    }
    const size_t at = ((size_t)seq * N + i) * kDM + head * kHD + lane * 4;
    if constexpr (kFlag) {
      unsigned long long* dst = static_cast<unsigned long long*>(att_any) + at;
      st_ll2(dst, __float_as_uint(o4.x), __float_as_uint(o4.y), tag_out);
      st_ll2(dst + 2, __float_as_uint(o4.z), __float_as_uint(o4.w), tag_out);
    } else {
      *reinterpret_cast<float4*>(static_cast<float*>(att_any) + at) = o4;
    }
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------
// Tail: per token LayerNorm(128) + ReLU + Linear(128->9), then the DDPM arithmetic.
// ---------------------------------------------------------------------------------------------
template <bool kFlag>
__device__ __forceinline__ void tail_token(const DenoiserDev& W, const DenoiserRun& R, int s, int t, bool last_step, unsigned tag_u,
                                           unsigned tag_x) {
  const int lane = threadIdx.x & 31;
  float4 v;
  if constexpr (kFlag) v = ld_ll_f4(R.fu + (size_t)s * kHid + lane * 4, tag_u);
  else v = __ldcg(reinterpret_cast<const float4*>(R.u + (size_t)s * kHid) + lane);
  const float mean = warp_sum(v.x + v.y + v.z + v.w) * (1.0f / kHid);
  v.x -= mean; v.y -= mean; v.z -= mean; v.w -= mean;
  const float rstd = 1.0f / sqrtf(warp_sum(v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w) * (1.0f / kHid) + kLnEps);
  const float4 g = __ldg(reinterpret_cast<const float4*>(W.ln_last_g) + lane);
  const float4 b = __ldg(reinterpret_cast<const float4*>(W.ln_last_b) + lane);
  v.x = fmaxf(v.x * rstd * g.x + b.x, 0.f);
  v.y = fmaxf(v.y * rstd * g.y + b.y, 0.f);
  v.z = fmaxf(v.z * rstd * g.z + b.z, 0.f);
  v.w = fmaxf(v.w * rstd * g.w + b.w, 0.f);
  float mine = 0.f;
#pragma unroll
  for (int c = 0; c < kTargetDim; ++c) {
    const float4 w = __ldg(reinterpret_cast<const float4*>(W.w_last3 + c * kHid) + lane);
    const float dot = warp_sum(w.x * v.x + w.y * v.y + w.z * v.z + w.w * v.w);
    if (lane == c) mine = dot + __ldg(W.b_last3 + c);
  }
  if (lane < kTargetDim) {
    const float* sc = W.sched + t * 8;
    const size_t e = (size_t)s * kTargetDim + lane;
    const float xt = __ldcg(R.x + e);
    const float x0 = sc[0] * xt - sc[1] * mine;             // predict_start_from_noise (:190-194)
    const float mu = sc[2] * x0 + sc[3] * xt;               // q_posterior mean (:201-205)
    float out = mu;
    const int k = (kT - 1) - t;                              // loop iteration index -> draw slot 1 + k
    if (t >= R.guide_below && t > 0 && R.draws) out = mu + sc[4] * __ldg(R.draws + (size_t)(1 + k) * R.tokens * kTargetDim + e);
    R.x[e] = out;
    if constexpr (kFlag) st_ll(R.fx + (size_t)s * 16 + lane, __float_as_uint(out), tag_x);  // what the next step of this launch reads
    if (R.trail && t >= R.guide_below) R.trail[(size_t)(1 + k) * R.tokens * kTargetDim + e] = out;
    if (last_step) {
      if (R.eps_out) R.eps_out[e] = mine;
      if (R.x0_out) R.x0_out[e] = x0;
      if (R.mean_out) R.mean_out[e] = mu;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// The persistent kernel
// ---------------------------------------------------------------------------------------------
template <int TS, bool kFlag>
__global__ void __launch_bounds__(kDenThreads, 1)
denoiser_kernel(const __grid_constant__ DenoiserDev W, const __grid_constant__ DenoiserRun R) {
#ifdef PDB_EMU  // tests/host/cuda_emu.h (CPU emulation of this kernel, test harness only): dynamic shared memory of this CTA
  float* const smem = reinterpret_cast<float*>(emu::g_cta->smem);
#else
  extern __shared__ __align__(16) float smem[];
#endif
  float* Xs = smem;  // [TS][K<=1024] or attention scratch
  __shared__ float pivot[32];
  __shared__ float xrow[32 * kTargetDim];
  const int S = R.tokens;
  const int tiles = (S + TS - 1) / TS;
  const int G = gridDim.x;
  unsigned bar_count = 0;
  long long clk[5] = {0, 0, 0, 0, 0};  // stage timing probe (thread 0, only with R.dbg_clock)
  const bool probe = R.dbg_clock != nullptr && threadIdx.x == 0;
  // Group barrier (kFlag = false only): release by one thread after the block barrier (cumulative over the CTA's writes),
  // acquire polls.  With flag-carrying activations the stages need none.
  auto barrier = [&]() {
    if constexpr (!kFlag) {
      ++bar_count;
      long long c0 = 0;
      if (probe) c0 = clock64();
      __syncthreads();
      if (threadIdx.x == 0) {
        red_release_add_u32(R.bar, 1u);
        while (ld_acquire_u32(R.bar) < bar_count * (unsigned)G) {
        }
      }
      __syncthreads();
      if (probe) clk[0] += clock64() - c0;
    }
  };
  // One linear stage: Y = epi(X' W^T + ...), work items = (token tile, 8-feature group).  The weights of this CTA's first
  // item are requested BEFORE the activations are waited for (barrier or tag poll), so their L2 latency hides behind the wait.
  auto linear_stage = [&](auto ktag, const float4* Wp, int O, auto&& load_x, const LinEpi& E, bool need_barrier) {
    constexpr int K = decltype(ktag)::value;
    const int groups = O / kFPI;
    const int n_items = tiles * groups;
    LinW<K> wreg;
    int item = blockIdx.x;
    if (item < n_items) linear_prefetch<K>(wreg, Wp, O, (item % groups) * kFPI);
    if (need_barrier) barrier();
    float* red = Xs + TS * K;
    int staged_tile = -1;  // the activations of a token tile are staged once and reused by this CTA's later items of the stage
    for (; item < n_items; item += G) {
      const int tt = item / groups, fg = item - tt * groups;
      if (item != (int)blockIdx.x) linear_prefetch<K>(wreg, Wp, O, fg * kFPI);
      long long c0 = 0, c1 = 0;
      if (probe) c0 = clock64();
      if (tt != staged_tile) {
        load_x(tt);
        staged_tile = tt;
      }
      __syncthreads();
      if (probe) c1 = clock64();
      linear_item<TS, K, kFlag>(wreg, Xs, red, fg * kFPI, E, tt * TS, S);
      if (probe) {
        clk[1] += c1 - c0;
        clk[2] += clock64() - c1;
      }
    }
  };
  // activation buffers of this instantiation, and the loader of a [tile, K] slab of one of them
  void* const h_buf = kFlag ? static_cast<void*>(R.fh) : static_cast<void*>(R.h);
  void* const att_buf = kFlag ? static_cast<void*>(R.fatt) : static_cast<void*>(R.att);
  void* const ff_buf = kFlag ? static_cast<void*>(R.fff) : static_cast<void*>(R.ff);
  void* const u_buf = kFlag ? static_cast<void*>(R.fu) : static_cast<void*>(R.u);
  auto load_tile = [&](auto ktag, const void* src, int tt, unsigned tag, const float* g, const float* b) {
    constexpr int K = decltype(ktag)::value;
    if constexpr (kFlag) load_rows_flag<K, TS>(Xs, static_cast<const unsigned long long*>(src), tt * TS, S, tag, g, b);
    else load_rows<K, TS>(Xs, static_cast<const float*>(src), tt * TS, S, g, b);
  };
  using KDM = std::integral_constant<int, kDM>;
  using KFF = std::integral_constant<int, kFF>;
  bool pending = false;  // a stage has written global activations that the next stage must wait for
  // ---- loop-invariant: zproj = z @ Wz^T + b_first + pivot * w_pivot   (denoiser.py:62-70); plain floats in both
  // instantiations: only the thread that wrote an element reads it again (epilogue of `first`, same item mapping) ----
  if (R.compute_zproj) {
    const LinEpi E = {W.b_first, nullptr, 0, false, nullptr, W.w_first_pivot, pivot, R.zproj, kDM, false, kEpiNone, 0u};
    linear_stage(std::integral_constant<int, kZ>{}, W.w_first_z, kDM,
                 [&](int tt) {
                   load_rows<kZ, TS>(Xs, R.z, tt * TS, S, nullptr, nullptr);
                   if (threadIdx.x < TS) pivot[threadIdx.x] = ((tt * TS + threadIdx.x) % R.frames == 0) ? 1.f : 0.f;
                 },
                 E, false);
    pending = true;
  }
  for (int t = R.t_hi; t >= R.t_lo; --t) {
    const unsigned v0 = R.tag_base + (unsigned)(R.t_hi - t) * kTagsPerStep;  // version ids of this step: v0 + id
    // ---- embed + first ----
    {
      const bool shadow = kFlag && t != R.t_hi;  // x of the previous step of THIS launch: flag-carrying shadow, version 42
      const LinEpi E = {nullptr, R.zproj, kDM, false, W.tproj + t * kDM, nullptr, nullptr, h_buf, kDM, kFlag, kEpiNone, v0};
      linear_stage(std::integral_constant<int, kPoseEmbPad>{}, W.w_first_x, kDM,
                   [&](int tt) { load_pose_embed(Xs, xrow, R.x, shadow ? R.fx : nullptr, v0 - kTagsPerStep + 42, tt * TS, TS, S); }, E,
                   pending);
    }
    pending = true;
    for (int l = 0; l < kLayers; ++l) {
      const LayerWeights& L = W.layer[l];
      const unsigned v_h_in = v0 + (l == 0 ? 0 : 5 * l), v_qkv = v0 + 1 + 5 * l, v_att = v0 + 2 + 5 * l, v_h_mid = v0 + 3 + 5 * l,
                     v_ff = v0 + 4 + 5 * l, v_h_out = v0 + 5 + 5 * l;
      void* const qkv_buf = kFlag ? static_cast<void*>(R.fqkv + (size_t)(l & 1) * S * 3 * kDM) : static_cast<void*>(R.qkv);
      // LN1 + QKV projection
      {
        const LinEpi E = {L.b_qkv, nullptr, 0, false, nullptr, nullptr, nullptr, qkv_buf, 3 * kDM, kFlag, kEpiNone, v_qkv};
        linear_stage(KDM{}, L.w_qkv, 3 * kDM, [&](int tt) { load_tile(KDM{}, h_buf, tt, v_h_in, L.ln1_g, L.ln1_b); }, E, true);
      }
      // attention per (sequence, head)
      barrier();
      {
        long long c0 = 0;
        if (probe) c0 = clock64();
        const int chunks = (R.frames + kDenWarps - 1) / kDenWarps;
        for (int item = blockIdx.x; item < R.batch * kHeads * chunks; item += G)
          attention_item<kFlag>(Xs, qkv_buf, att_buf, item / (kHeads * chunks), (item / chunks) % kHeads, item % chunks, R.frames,
                                v_qkv, v_att);
        if (probe) clk[3] += clock64() - c0;
      }
      // out-proj + residual (in place on h: each element is read and written by the same thread)
      {
        const LinEpi E = {L.b_out, h_buf, kDM, kFlag, nullptr, nullptr, nullptr, h_buf, kDM, kFlag, kEpiNone, v_h_mid};
        linear_stage(KDM{}, L.w_out, kDM, [&](int tt) { load_tile(KDM{}, att_buf, tt, v_att, nullptr, nullptr); }, E, true);
      }
      // LN2 + FF1 + ReLU
      {
        const LinEpi E = {L.b_ff1, nullptr, 0, false, nullptr, nullptr, nullptr, ff_buf, kFF, kFlag, kEpiRelu, v_ff};
        linear_stage(KDM{}, L.w_ff1, kFF, [&](int tt) { load_tile(KDM{}, h_buf, tt, v_h_mid, L.ln2_g, L.ln2_b); }, E, true);
      }
      // FF2 + residual
      {
        const LinEpi E = {L.b_ff2, h_buf, kDM, kFlag, nullptr, nullptr, nullptr, h_buf, kDM, kFlag, kEpiNone, v_h_out};
        linear_stage(KFF{}, L.w_ff2, kDM, [&](int tt) { load_tile(KFF{}, ff_buf, tt, v_ff, nullptr, nullptr); }, E, true);
      }
    }
    // last0: Linear(512 -> 128)
    {
      const LinEpi E = {W.b_last0, nullptr, 0, false, nullptr, nullptr, nullptr, u_buf, kHid, kFlag, kEpiNone, v0 + 41};
      linear_stage(KDM{}, W.w_last0, kHid, [&](int tt) { load_tile(KDM{}, h_buf, tt, v0 + 5 * kLayers, nullptr, nullptr); }, E, true);
    }
    // tail: one warp per token
    barrier();
    {
      long long c0 = 0;
      if (probe) c0 = clock64();
      const int warp_global = blockIdx.x * kDenWarps + (threadIdx.x >> 5);
      for (int s = warp_global; s < S; s += G * kDenWarps) tail_token<kFlag>(W, R, s, t, t == R.t_lo, v0 + 41, v0 + 42);
      if (probe) clk[4] += clock64() - c0;
    }
    pending = true;
  }
  if (probe) {
    long long* c = R.dbg_clock + (size_t)blockIdx.x * 8;
    for (int k = 0; k < 5; ++k) c[k] += clk[k];
    c[5] += R.t_hi - R.t_lo + 1;
  }
}

inline size_t denoiser_smem_bytes(int TS, int frames) {
  size_t lin = (size_t)TS * kFF + (size_t)kDenWarps * TS * kFPI;                      // X tile + reduction
  size_t att = (size_t)frames * (kHD + 4) + (size_t)frames * kHD + 2 * kDenWarps * kHD;  // K, V, Q, P
  return sizeof(float) * (lin > att ? lin : att) + 256;
}

}  // namespace pdb
